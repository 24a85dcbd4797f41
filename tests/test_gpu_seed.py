"""seeddot_nll (SEED-Encoder) on the sm_90a encoder, in fp16 and bf16: embeddings against the reference's golden ones
(tests/golden/encoder_seed.npz), the packed path against the dense one, whole-model gradients against autograd of the
SEED oracle (oracle/seed_oracle.py), packed training, the config's dropout rates, Lamb and the unused classification
heads, and an end-to-end refresh through run_ann_data_gen."""
import json
import os
import random

import numpy as np
import pytest
import torch

from ance_b200 import _lib
from ance_b200.models import SEEDEncoderConfig, SEEDEncoderDot_NLL_LN_B200
from ance_b200.synthetic import random_seed_state_dict, write_marco_like_dir, write_seed_checkpoint
from oracle import flat_ip_oracle, refresh_oracle
from oracle.seed_oracle import SEEDDotOracle

pytestmark = pytest.mark.gpu

FMTS = ["fp16", "bf16"]
GOLD = os.path.join(os.path.dirname(__file__), "golden")
P = "seed_encoder.encoder.sentence_encoder."
# the embedding gate of README.md / tests/test_gpu_encoder.py; the bf16 storage variant is held to max |diff| <= 0.1
# there (one bf16 rounding of a value in [4, 8) is already 0.0156)
COS_GATE, ABS_GATE = 0.9995, {"fp16": 0.03, "bf16": 0.1}
# per-tensor gradient gate of tests/test_gpu_encoder_backward.py (fp16 / bf16 forward)
GATE = {"fp16": 0.03, "bf16": 0.05}


def _model(fmt, n_layer, vocab, seed, **cfg):
    m = SEEDEncoderDot_NLL_LN_B200(SEEDEncoderConfig(encoder_layers=n_layer, vocab_size=vocab, **cfg))
    m.load_state_dict(random_seed_state_dict(seed=seed, n_layer=n_layer, vocab=vocab))
    m.encoder_operand = fmt
    return m.cuda().eval()


def _no_tf32():
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    return prev


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLD, "encoder_seed.npz"))


@pytest.mark.parametrize("fmt", FMTS)
def test_embeddings_match_the_reference(golden, fmt):
    m = _model(fmt, 12, 32769, int(golden["seed"]))
    for key in ("p", "q", "f"):
        ids = torch.from_numpy(golden[key + "ids"]).cuda()
        ref = torch.from_numpy(golden[key + "emb"])
        with torch.no_grad():
            out = m.body_emb(ids, None).cpu()
            # attention_mask is ignored: the mask comes from ids != pad_token_id
            noise = torch.randint(0, 2, ids.shape, device="cuda")
            assert torch.equal(m.query_emb(ids, noise).cpu(), out)
            assert torch.equal(m(ids, noise).cpu(), out)
            packed = m.body_emb_packed(ids, align=16).cpu()
            dense1 = m.query_emb_packed(ids, align=1).cpu()
        m.check_inputs()
        cos = torch.nn.functional.cosine_similarity(out, ref, dim=-1).min().item()
        err = (out - ref).abs().max().item()
        print(f"seeddot_nll {fmt} {key}: min cosine {cos:.6f}, max |diff| {err:.4f}")
        assert cos >= COS_GATE and err <= ABS_GATE[fmt], (key, cos, err)
        assert torch.equal(packed, out), key                       # align 16: bit-identical to the dense forward
        # align 1 sums in another order; through 12 layers of 16-bit storage that is held to the same gate
        cos1 = torch.nn.functional.cosine_similarity(dense1, ref, dim=-1).min().item()
        assert cos1 >= COS_GATE and (dense1 - ref).abs().max().item() <= ABS_GATE[fmt], key
    # the triplet loss of NLL.forward
    q, a, b = (torch.from_numpy(x).cuda() for x in (golden["qids"][:3], golden["pids"][:3], golden["pids"][3:]))
    with torch.no_grad():
        (loss,) = m(q, None, a, None, b, None)
    # logits are dot products of two 768-wide LayerNorm outputs, so the loss carries both embeddings' error: 2 % of its
    # value for fp16 storage, 5 % for bf16 (8 significant bits instead of 11; measured 2.1 % at 12 layers)
    tol = {"fp16": 0.02, "bf16": 0.05}[fmt]
    assert abs(float(loss) - float(golden["loss"])) <= tol * abs(float(golden["loss"])), (float(loss), golden["loss"])


def test_dimensions_the_kernels_reject():
    m = SEEDEncoderDot_NLL_LN_B200(SEEDEncoderConfig(encoder_layers=1, vocab_size=100, encoder_attention_heads=16))
    m = m.cuda()
    with pytest.raises(_lib.AnceError, match="head_dim must be 64"):
        m.query_emb(torch.full((1, 8), 5, device="cuda"))


def _triplet():
    g = np.load(os.path.join(GOLD, "seed_grads.npz"))
    return g, [torch.from_numpy(g[k]).cuda() for k in ("q_ids", "a_ids", "b_ids")]


def _oracle_grads(sd, n_layer, batches):
    prev = _no_tf32()
    try:
        orc = SEEDDotOracle(sd, n_layer=n_layer, device="cuda")
        leaves = orc.leaves()
        loss = orc.nll_loss(*batches)
        loss.backward()
        return orc, float(loss.detach()), {k: v.grad for k, v in leaves.items()}
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


def _compare_grads(model, gref, fmt, name, extra=0.0):
    """Every parameter's gradient within GATE of the oracle's, relative to its norm; the key biases (exact gradient
    zero) relative to the query bias's.  The classification heads take no gradient."""
    bad, rels = [], {}
    for k, p in model.named_parameters():
        if k.startswith("classification_heads."):
            assert p.grad is None, k
            continue
        ref = gref[k]
        if k.endswith("self_attn.k_proj.bias"):
            rel = float(p.grad.norm() / gref[k.replace("k_proj", "q_proj")].norm())
        else:
            rel = float((p.grad - ref).norm() / ref.norm().clamp_min(1e-30))
        rels[k] = rel
        if not rel <= GATE[fmt] + extra:
            bad.append((k, rel))
    worst = max(rels, key=rels.get)
    print(f"{name} {fmt}: worst per-tensor relative error {rels[worst]:.4f} ({worst}; gate {GATE[fmt] + extra:.4f})")
    assert not bad, f"{name} {fmt}: {bad}"


@pytest.mark.parametrize("fmt", FMTS)
def test_triplet_gradients_match_the_oracle(fmt):
    g, (q, a, b) = _triplet()
    sd = random_seed_state_dict(seed=int(g["seed"]), n_layer=2, vocab=1000)
    m = _model(fmt, 2, 1000, int(g["seed"])).set_trainable(True)
    (loss,) = m(q, torch.ones_like(q), a, torch.zeros_like(a), b, None)
    assert loss.grad_fn is not None
    loss.backward()
    orc, lref, gref = _oracle_grads(sd, 2, (q, a, b))
    assert abs(lref - float(g["loss"])) <= 1e-4 * abs(lref)
    assert abs(float(loss.detach()) - lref) <= 0.02 * abs(lref), (float(loss.detach()), lref)
    # dL/d(embeddings) carries each side's forward error: widen the gate by twice its relative error (as the rdot_nll
    # triplet test does)
    with torch.no_grad():
        ours = [m.query_emb(q), m.body_emb(a), m.body_emb(b)]
        prev = _no_tf32()
        try:
            theirs = [orc.query_emb(x) for x in (q, a, b)]
        finally:
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
    up = []
    for es in (ours, theirs):
        leaves = [e.detach().clone().requires_grad_(True) for e in es]
        lm = torch.stack([(leaves[0] * leaves[1]).sum(-1), (leaves[0] * leaves[2]).sum(-1)], dim=1)
        (-torch.log_softmax(lm, dim=1)[:, 0]).mean().backward()
        up.append(torch.cat([x.grad.reshape(-1) for x in leaves]))
    rel_up = float((up[0] - up[1]).norm() / up[1].norm())
    print(f"seeddot_nll triplet {fmt}: upstream gradient relative error {rel_up:.4f}")
    _compare_grads(m, gref, fmt, "seeddot_nll triplet", extra=2 * rel_up)
    # nn.Embedding(padding_idx=pad_token_id) for tokens and positions: no gradient in those rows
    assert not m.get_parameter(P + "embed_tokens.weight").grad[1].any()
    assert not m.get_parameter(P + "embed_positions.weight").grad[1].any()
    assert m.get_buffer(P + "type_row").grad is None and not m.get_buffer(P + "type_row").any()


def _holed_batch(B, L, seed, vocab=1000):
    gen = np.random.default_rng(seed)
    lens = gen.integers(4, L + 1, size=B)
    lens[0] = L
    ids = np.full((B, L), 1, dtype=np.int64)
    for i, n in enumerate(lens):
        ids[i, :n] = gen.integers(3, vocab, size=n)
        ids[i, 0] = 0
    ids[1, min(3, lens[1] - 2)] = 1   # a pad id inside a row: that row takes the dense path
    return torch.from_numpy(ids).cuda()


@pytest.mark.parametrize("fmt", FMTS)
def test_packed_training_equals_dense(fmt):
    batches = [_holed_batch(4, 64, 1), _holed_batch(4, 512, 2), _holed_batch(4, 512, 3)]
    res = []
    for packed in (False, True):
        m = _model(fmt, 2, 1000, 4).set_trainable(True, max_len=512, packed=packed)
        (loss,) = m(*[x for t in batches for x in (t, None)])
        loss.backward()
        with torch.no_grad():
            embs = [m.body_emb(t) for t in batches]
        res.append((float(loss.detach()), {k: p.grad for k, p in m.named_parameters() if p.grad is not None}, embs))
    (l0, g0, e0), (l1, g1, e1) = res
    assert all(torch.equal(x, y) for x, y in zip(e0, e1))
    assert l0 == l1
    assert set(g0) == set(g1) and not any(k.startswith("classification_heads.") for k in g0)
    worst = 0.0
    for k in g0:
        if k.endswith("k_proj.bias"):
            rel = float((g1[k] - g0[k]).norm() / g0[k.replace("k_proj", "q_proj")].norm())
        else:
            rel = float((g1[k] - g0[k]).norm() / g0[k].norm().clamp_min(1e-30))
        worst = max(worst, rel)
        assert rel <= 1e-4, (k, rel)
    print(f"seeddot_nll packed training {fmt}: worst relative gradient difference to dense {worst:.2e}")


def test_dropout_uses_the_config_rates():
    m = _model("fp16", 2, 1000, 4, dropout=0.2, attention_dropout=0.05)
    m.set_trainable(True, max_len=128, dropout=True)
    assert m._dropout == (0.2, 0.05)
    ids = _holed_batch(6, 128, 5)
    m.train()
    torch.manual_seed(7)
    out = m.query_emb(ids)
    torch.manual_seed(7)
    lo, hi = torch.randint(0, 2 ** 32, (2,), dtype=torch.int64).tolist()
    enc = m._encoder(ids.device)
    i32 = ids.to(torch.int32).contiguous()
    ref, _ = enc.forward_train(i32, None, (i32 != 1).to(torch.uint8), (0.2, 0.05, lo | (hi << 32)))
    assert torch.equal(out.detach(), ref)
    out.sum().backward()
    m.eval()
    with torch.no_grad():
        assert not torch.equal(m.query_emb(ids), ref)


def test_lamb_leaves_the_classification_heads_untouched():
    from ance_b200.optim import Lamb
    m = _model("fp16", 2, 1000, 4).set_trainable(True)
    heads = {k: p.detach().clone() for k, p in m.named_parameters() if k.startswith("classification_heads.")}
    rest = {k: p.detach().clone() for k, p in m.named_parameters() if not k.startswith("classification_heads.")}
    opt = Lamb(m.parameters(), lr=1e-3, weight_decay=0.01)
    q, a, b = _holed_batch(4, 32, 6), _holed_batch(4, 128, 7), _holed_batch(4, 128, 8)
    m.train()
    (loss,) = m(q, None, a, None, b, None)
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    for k, p in m.named_parameters():
        if k in heads:
            assert p.grad is None and torch.equal(p.detach(), heads[k]), k
            assert not opt.state[p], k
        elif k not in (P + "embed_tokens.weight", P + "embed_positions.weight"):
            assert not torch.equal(p.detach(), rest[k]), k


def test_refresh_end_to_end(tmp_path):
    """run_ann_data_gen --model_type seeddot_nll --max_seq_length 512 on a synthetic checkpoint and MARCO-like data: the
    packed exact path and --no_varlen write the same files, and they follow from embeddings whose top-k matches the
    oracle's."""
    from ance_b200.drivers import run_ann_data_gen as drv
    vocab, n_layer = 32769, 2
    data, ck = tmp_path / "data", tmp_path / "init_model"
    write_marco_like_dir(str(data), 1500, 120, 40, L_p=512, L_q=64, seed=2, vocab=vocab)
    write_seed_checkpoint(str(ck), seed=9, n_layer=n_layer, vocab=vocab)

    def argv(out, *extra):
        return ["--data_dir", str(data), "--training_dir", str(tmp_path / "no_training_dir_yet"), "--init_model_dir",
                str(ck), "--model_type", "seeddot_nll", "--output_dir", str(out), "--cache_dir", str(tmp_path / "cache"),
                "--end_output_num", "0", "--max_seq_length", "512", "--max_query_length", "64",
                "--per_gpu_eval_batch_size", "16", "--topk_training", "20", "--negative_sample", "5",
                "--ann_chunk_factor", "1", "--reference_sampling", "--seed", "0", *extra]

    outs = {}
    for name, extra in (("packed", ()), ("dense", ("--no_varlen",))):
        out = tmp_path / name
        drv.main(argv(out, *extra))
        outs[name] = {f: open(out / f, "rb").read() for f in ("ann_training_data_0", "ann_ndcg_0")}
    assert outs["packed"] == outs["dense"]
    ndcg = json.loads(outs["packed"]["ann_ndcg_0"])
    assert ndcg["checkpoint"] == str(ck) and 0.0 <= ndcg["ndcg"] <= 1.0
    # the oracle pipeline downstream of the same GPU embeddings reproduces the training file
    args = drv.get_arguments(argv(tmp_path / "packed"))
    drv.set_env(args)
    _, _, model = drv.load_model(args, str(ck))
    assert type(model) is SEEDEncoderDot_NLL_LN_B200
    be = drv.B200Backend(args, model)
    assert be.mask_mode == "ids"
    emb = {k: be.encode(str(data / k), k != "passages") for k in ("passages", "train-query")}
    P_, p2id = emb["passages"][0].cpu().numpy(), emb["passages"][1]
    Q, q2id = emb["train-query"][0].cpu().numpy(), emb["train-query"][1]
    _, I = flat_ip_oracle.search(P_, Q, 20)
    train_pos = {}
    with open(data / "train-qrel.tsv") as f:
        for line in f:
            qq, pp, _ = line.split("\t")
            train_pos[int(qq)] = int(pp)
    rng = random.Random(0)
    negs, _, _ = refresh_oracle.generate_negatives(q2id, p2id, train_pos, I, set(q2id.tolist()), 5, False, rng)
    want = "".join(refresh_oracle.training_data_lines(q2id, train_pos, negs, set(q2id.tolist()), rng))
    assert outs["packed"]["ann_training_data_0"].decode() == want
    # those embeddings against the fp32 oracle's: top-20 overlap
    from ance_b200.data import EmbeddingCache
    sd = random_seed_state_dict(seed=9, n_layer=n_layer, vocab=vocab)
    prev = _no_tf32()
    try:
        orc = SEEDDotOracle(sd, n_layer=n_layer, device="cuda")
        ref = {}
        for k in ("passages", "train-query"):
            c = EmbeddingCache(str(data / k))
            ids = torch.from_numpy(np.asarray(c.memmap()["ids"]).astype(np.int64))
            with torch.no_grad():
                ref[k] = torch.cat([orc.body_emb(ids[s:s + 64].cuda()) for s in range(0, len(ids), 64)]).cpu().numpy()
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
    assert p2id.tolist() == list(range(len(p2id))) and q2id.tolist() == list(range(len(q2id)))
    _, I_ref = flat_ip_oracle.search(ref["passages"], ref["train-query"], 20)
    overlap = np.mean([len(set(I[i]) & set(I_ref[i])) / 20 for i in range(len(I))])
    print(f"seeddot_nll refresh: top-20 overlap with the oracle embeddings {overlap:.4f}")
    assert overlap >= 0.99
