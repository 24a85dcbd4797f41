"""Synthetic inputs of the ANN-refresh path in the reference's own formats (SURVEY.md §8d): seeded-random checkpoints
in the HF key layout, token caches (`passages`, `train-query`, `dev-query` + `_meta`), qrels.  There is no network in
the build / GPU boxes, hence no MS MARCO and no pretrained weights: bench.py, tools/full_refresh.py and the tests run
the real code path on data of the real SHAPE, and say so ("data": "synthetic").

Formats follow SURVEY.md Appendix B: record = big-endian int32 length + L native int32 ids
(data/msmarco_data.py:160-176,258,272 ; utils/util.py:264-283); qrels `qoff\\tpoff\\trel` (msmarco_data.py:116-121).
"""
from __future__ import annotations

import json
import os
from typing import Dict, Optional

import numpy as np
import torch


def random_roberta_state_dict(seed=0, n_layer=12, hidden=768, ffn=3072, vocab=50265, max_pos=514,
                              head=True, prefix="roberta.") -> Dict[str, torch.Tensor]:
    """Seeded random weights in the checkpoint's key layout (SURVEY.md §8 a2): what `save_pretrained` of the
    reference's RobertaDot_NLL_LN / the DPR BiEncoder halves would hold."""
    g = torch.Generator().manual_seed(seed)

    def n(*shape, std=0.02):
        return torch.randn(*shape, generator=g) * std

    sd = {
        prefix + "embeddings.word_embeddings.weight": n(vocab, hidden),
        prefix + "embeddings.position_embeddings.weight": n(max_pos, hidden),
        prefix + "embeddings.token_type_embeddings.weight": n(1 if prefix == "roberta." else 2, hidden),
        prefix + "embeddings.LayerNorm.weight": 1.0 + n(hidden, std=0.05),
        prefix + "embeddings.LayerNorm.bias": n(hidden, std=0.05),
    }
    for l in range(n_layer):
        lp = f"{prefix}encoder.layer.{l}."
        for nm in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense"):
            sd[lp + nm + ".weight"] = n(hidden, hidden, std=0.04)
            sd[lp + nm + ".bias"] = n(hidden, std=0.02)
        sd[lp + "intermediate.dense.weight"] = n(ffn, hidden, std=0.04)
        sd[lp + "intermediate.dense.bias"] = n(ffn, std=0.02)
        sd[lp + "output.dense.weight"] = n(hidden, ffn, std=0.04)
        sd[lp + "output.dense.bias"] = n(hidden, std=0.02)
        for nm in ("attention.output.LayerNorm", "output.LayerNorm"):
            sd[lp + nm + ".weight"] = 1.0 + n(hidden, std=0.05)
            sd[lp + nm + ".bias"] = n(hidden, std=0.05)
    if head:
        sd["embeddingHead.weight"] = n(768, hidden, std=0.04)
        sd["embeddingHead.bias"] = n(768, std=0.02)
        sd["norm.weight"] = 1.0 + n(768, std=0.05)
        sd["norm.bias"] = n(768, std=0.05)
    return sd


def roberta_base_config(**over):
    from transformers import RobertaConfig
    kw = dict(vocab_size=50265, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
              max_position_embeddings=514, type_vocab_size=1, layer_norm_eps=1e-5, pad_token_id=1, bos_token_id=0,
              eos_token_id=2)
    kw.update(over)
    return RobertaConfig(**kw)


def write_checkpoint(path: str, seed: int = 0, n_layer: int = 12, vocab: int = 50265) -> None:
    """`training_dir/checkpoint-N/`-style payload (run_ann.py:307-331): config.json + pytorch_model.bin."""
    os.makedirs(path, exist_ok=True)
    roberta_base_config(num_hidden_layers=n_layer, vocab_size=vocab).save_pretrained(path)
    torch.save(random_roberta_state_dict(seed=seed, n_layer=n_layer, vocab=vocab), os.path.join(path, "pytorch_model.bin"))


def random_seed_state_dict(seed=0, n_layer=12, hidden=768, ffn=3072, vocab=32769, max_pos=514,
                           num_labels=2) -> Dict[str, torch.Tensor]:
    """Seeded random weights of the reference's SEEDEncoderDot_NLL_LN (`seeddot_nll`) under its own parameter names and
    in its registration order: what its `save_pretrained` would hold.  max_pos = max_positions + pad_token_id + 1."""
    g = torch.Generator().manual_seed(seed)

    def n(*shape, std=0.02):
        return torch.randn(*shape, generator=g) * std

    p = "seed_encoder.encoder.sentence_encoder."
    sd = {p + "embed_tokens.weight": n(vocab, hidden), p + "embed_positions.weight": n(max_pos, hidden)}
    for l in range(n_layer):
        lp = f"{p}layers.{l}."
        for nm in ("self_attn.k_proj", "self_attn.v_proj", "self_attn.q_proj", "self_attn.out_proj"):
            sd[lp + nm + ".weight"] = n(hidden, hidden, std=0.04)
            sd[lp + nm + ".bias"] = n(hidden, std=0.02)
        sd[lp + "self_attn_layer_norm.weight"] = 1.0 + n(hidden, std=0.05)
        sd[lp + "self_attn_layer_norm.bias"] = n(hidden, std=0.05)
        sd[lp + "fc1.weight"] = n(ffn, hidden, std=0.04)
        sd[lp + "fc1.bias"] = n(ffn, std=0.02)
        sd[lp + "fc2.weight"] = n(hidden, ffn, std=0.04)
        sd[lp + "fc2.bias"] = n(hidden, std=0.02)
        sd[lp + "final_layer_norm.weight"] = 1.0 + n(hidden, std=0.05)
        sd[lp + "final_layer_norm.bias"] = n(hidden, std=0.05)
    sd[p + "emb_layer_norm.weight"] = 1.0 + n(hidden, std=0.05)
    sd[p + "emb_layer_norm.bias"] = n(hidden, std=0.05)
    sd["classification_heads.dense.weight"] = n(hidden, hidden, std=0.04)
    sd["classification_heads.dense.bias"] = n(hidden, std=0.02)
    sd["classification_heads.out_proj.weight"] = n(num_labels, hidden, std=0.04)
    sd["classification_heads.out_proj.bias"] = n(num_labels, std=0.02)
    sd["embeddingHead.weight"] = n(768, hidden, std=0.04)
    sd["embeddingHead.bias"] = n(768, std=0.02)
    sd["norm.weight"] = 1.0 + n(768, std=0.05)
    sd["norm.bias"] = n(768, std=0.05)
    return sd


def write_seed_checkpoint(path: str, seed: int = 0, n_layer: int = 12, vocab: int = 32769, **config) -> None:
    """A `seeddot_nll` checkpoint directory: config.json (SEEDEncoderConfig; `config` overrides its defaults) +
    pytorch_model.bin of random_seed_state_dict."""
    from .models import SEEDEncoderConfig
    os.makedirs(path, exist_ok=True)
    cfg = SEEDEncoderConfig(encoder_layers=n_layer, vocab_size=vocab, **config)
    cfg.save_pretrained(path)
    torch.save(random_seed_state_dict(seed=seed, n_layer=n_layer, hidden=cfg.encoder_embed_dim,
                                      ffn=cfg.encoder_ffn_embed_dim, vocab=vocab,
                                      max_pos=cfg.max_positions + cfg.pad_token_id + 1, num_labels=cfg.num_labels),
               os.path.join(path, "pytorch_model.bin"))


def write_token_cache(base_path: str, n: int, L: int, mean_len: float, sd_len: float, min_len: int, seed: int,
                      vocab: int = 50265, pad_id: int = 1, bos: int = 0, eos: int = 2, full_length: bool = False,
                      chunk: int = 1 << 18, part: int = 0, n_parts: int = 1) -> None:
    """`n` records of `L` tokens, written in chunks (the 8.84M-passage cache is 4.56 GB): lengths ~ clipped
    N(mean, sd) -> [min_len, L] (or all = L), ids uniform in [3, vocab), position 0 = <s>, last real token = </s>,
    right-padded with pad_id.  Deterministic in (seed, chunk): with n_parts > 1 several processes write disjoint chunks
    (chunk index % n_parts == part) of the same pre-sized file and the result is the one a single writer produces."""
    rec = np.dtype([("len", ">i4"), ("ids", "<i4", (L,))])
    if n_parts > 1 and not os.path.exists(base_path):
        raise FileNotFoundError(base_path + ": with n_parts > 1 the file must be created (truncated to size) first")
    with open(base_path, "r+b" if n_parts > 1 else "wb") as f:
        for ci, c0 in enumerate(range(0, n, chunk)):
            if ci % n_parts != part:
                continue
            f.seek(c0 * rec.itemsize)
            m = min(chunk, n - c0)
            rng = np.random.default_rng([seed, c0])
            lens = np.full(m, L, dtype=np.int64) if full_length else \
                np.clip(rng.normal(mean_len, sd_len, size=m).round().astype(np.int64), min_len, L)
            ids = rng.integers(3, vocab, size=(m, L), dtype=np.int32)
            ids[np.arange(L)[None, :] >= lens[:, None]] = pad_id
            ids[:, 0] = bos
            ids[np.arange(m), lens - 1] = eos
            out = np.empty(m, dtype=rec)
            out["len"] = lens
            out["ids"] = ids
            out.tofile(f)
    if part == 0:
        with open(base_path + "_meta", "w") as f:
            json.dump({"type": "int32", "total_number": int(n), "embedding_size": int(L)}, f)


def presize_token_cache(base_path: str, n: int, L: int) -> None:
    with open(base_path, "wb") as f:
        f.truncate(n * (4 + 4 * L))


def write_marco_like_dir(data_dir: str, n_passages: int, n_train_queries: int, n_dev_queries: int, L_p: int = 128,
                         L_q: int = 64, seed: int = 0, full_length_passages: bool = False, vocab: int = 50265,
                         part: int = 0, n_parts: int = 1, barrier=None) -> None:
    """The refresher's `--data_dir` (run_ann_data_gen.py:78-98,236-263): three token caches + train / dev qrels with one
    random positive per query (SURVEY.md §8d cfg 1-3).  n_parts > 1: called by every rank of a job with its own `part`
    and a `barrier` callable; the ranks share the writing of the caches."""
    os.makedirs(data_dir, exist_ok=True)
    specs = [("passages", n_passages, L_p, 76, 28, 8, seed + 1, full_length_passages),
             ("train-query", n_train_queries, L_q, 9, 3, 4, seed + 2, False),
             ("dev-query", n_dev_queries, L_q, 9, 3, 4, seed + 3, False)]
    if n_parts > 1:
        if part == 0:
            for name, n, L, *_ in specs:
                presize_token_cache(os.path.join(data_dir, name), n, L)
        barrier()
    for name, n, L, mean, sd, lo, sd_seed, full in specs:
        write_token_cache(os.path.join(data_dir, name), n, L, mean, sd, lo, sd_seed, vocab, full_length=full, part=part,
                          n_parts=n_parts)
    if part != 0:
        return
    rng = np.random.default_rng(seed + 4)
    pos = rng.integers(0, n_passages, size=n_train_queries)
    with open(os.path.join(data_dir, "train-qrel.tsv"), "w") as f:
        f.write("".join("%d\t%d\t1\n" % (q, p) for q, p in enumerate(pos.tolist())))
    pos = rng.integers(0, n_passages, size=n_dev_queries)
    with open(os.path.join(data_dir, "dev-qrel.tsv"), "w") as f:
        f.write("".join("%d\t%d\t1\n" % (q, p) for q, p in enumerate(pos.tolist())))


def synth_index_rows(n: int, dim: int, dev, seed: int, kind: str = "layernorm_clustered", chunk: int = 1 << 20,
                     centroids: Optional[torch.Tensor] = None):
    """Chunks of synthetic index rows generated on the device (SURVEY.md §8d):
      layernorm_clustered  z ~ N(0, I) mixed 0.5 / 0.5 with one of 1024 centroids, each row standardised to mean 0 /
                           variance 1 (|row| = sqrt(dim): what the head's LayerNorm emits)               cfg 2-4
      dpr                  un-normalised: 0.5 * N(0, I) + a shared offset (BERT CLS anisotropy), row norms vary  cfg 5
      iid                  standardised N(0, I) rows, no structure (smallest score gaps)
      heavy_tail           layernorm_clustered rows scaled by a log-normal factor (sigma 0.35)
      near_duplicate       layernorm_clustered where every row has ~8 copies perturbed by 1e-3"""
    g = torch.Generator(device=dev).manual_seed(seed)
    if centroids is None:
        centroids = torch.randn(1024, dim, device=dev, generator=torch.Generator(device=dev).manual_seed(7))
    offset = torch.randn(dim, device=dev, generator=torch.Generator(device=dev).manual_seed(8)) * 0.3

    def ln(x):
        return (x - x.mean(1, keepdim=True)) / x.std(1, keepdim=True, unbiased=False)

    for s in range(0, n, chunk):
        m = min(chunk, n - s)
        if kind == "dpr":
            yield 0.5 * torch.randn(m, dim, device=dev, generator=g) + offset
            continue
        if kind == "iid":
            yield ln(torch.randn(m, dim, device=dev, generator=g))
            continue
        base_n = (m + 7) // 8 if kind == "near_duplicate" else m
        x = 0.5 * torch.randn(base_n, dim, device=dev, generator=g) + \
            0.5 * centroids[torch.randint(0, centroids.shape[0], (base_n,), device=dev, generator=g)]
        x = ln(x)
        if kind == "near_duplicate":
            x = x.repeat_interleave(8, dim=0)[:m]
            x = x + 1.0e-3 * torch.randn(m, dim, device=dev, generator=g)
        elif kind == "heavy_tail":
            x = x * torch.exp(0.35 * torch.randn(m, 1, device=dev, generator=g))
        yield x
