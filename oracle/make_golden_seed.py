"""Generate tests/golden/encoder_seed.npz and tests/golden/seed_grads.npz by running the REFERENCE's own
SEEDEncoderDot_NLL_LN (model/models.py:201-221, model/SEED_Encoder/) on CPU in fp32.

Run in the build container only (the GPU machine has no reference checkout):

    python oracle/make_golden_seed.py

Under transformers 5.x the reference's constructor fails in PreTrainedModel.init_weights -> tie_weights (its
SEEDEncoderModel has no `all_tied_weights_keys`).  init_weights only draws initial values, which the seeded state dict
below overwrites, so it is replaced by a no-op before the import.

encoder_seed.npz (12 layers, vocabulary 32769, random_seed_state_dict(seed=0)):
  param_names          the reference's named_parameters() order
  pids / pemb          6 passages of L = 512: full rows with no padding, prefix padding, a pad id inside a full row and
                       inside a padded one
  qids / qemb          6 queries of L = 64, the same kinds
  fids / femb          4 queries of L = 64 padded with id 0, which is not pad_token_id (1): the reference attends to them
  loss                 NLL.forward's triplet loss of (qids[:3], pids[:3], pids[3:])
seed_grads.npz (2 layers, vocabulary 1000, random_seed_state_dict(seed=1)):
  q_ids, a_ids, b_ids  the triplet (4 x 32, 4 x 128, 4 x 128; prefix padding and one pad id inside a row)
  loss                 NLL.forward's loss
  names, sketch        per parameter with a gradient: oracle.seed_oracle.grad_sketch (norm + 4 seeded projections)
  tok_pad_row, pos_pad_row   the embed_tokens / embed_positions gradient rows at pad_token_id (nn.Embedding padding_idx)
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)

from oracle.seed_oracle import SEEDDotOracle, grad_sketch, random_seed_state_dict  # noqa: E402

PAD = 1


def reference_seed_model(n_layer, vocab, sd):
    sys.path.append(REF)
    for m in ("pytrec_eval", "faiss", "tensorboardX"):
        sys.modules.setdefault(m, types.ModuleType(m))
    sys.modules["tensorboardX"].SummaryWriter = object
    import transformers
    transformers.__dict__.setdefault("AdamW", torch.optim.AdamW)
    from transformers.modeling_utils import PreTrainedModel
    PreTrainedModel.init_weights = lambda self: None
    import model.models as M
    from model.SEED_Encoder import SEEDEncoderConfig

    cfg = SEEDEncoderConfig(encoder_layers=n_layer, vocab_size=vocab, num_labels=2, dropout=0.0, attention_dropout=0.0)
    ref = M.SEEDEncoderDot_NLL_LN(cfg)
    ref.load_state_dict(sd, strict=True)
    return ref.eval()


def make_ids(rng, lens, L, vocab, pad=PAD, holes=()):
    """Rows of lens[b] tokens (<s>=0 first, </s>=2 last) right-padded with `pad`; (row, col) in holes gets pad_token_id."""
    ids = np.full((len(lens), L), pad, dtype=np.int32)
    for b, n in enumerate(lens):
        ids[b, :n] = rng.integers(3, vocab, size=n)
        ids[b, 0], ids[b, n - 1] = 0, 2
    for r, c in holes:
        ids[r, c] = PAD
    return ids


def golden_embeddings():
    rng = np.random.default_rng(0)
    vocab = 32769
    sd = random_seed_state_dict(seed=0, n_layer=12, vocab=vocab)
    ref = reference_seed_model(12, vocab, sd)
    names = [n for n, _ in ref.named_parameters()]
    assert names == list(sd), "random_seed_state_dict is not in the reference's order"
    pids = make_ids(rng, [512, 300, 77, 512, 130, 9], 512, vocab, holes=[(3, 200), (4, 50)])
    qids = make_ids(rng, [64, 12, 33, 5, 64, 20], 64, vocab, holes=[(4, 10), (5, 7)])
    fids = make_ids(rng, [64, 30, 8, 17], 64, vocab, pad=0)
    orc = SEEDDotOracle(sd, n_layer=12)
    out = {"seed": np.int64(0), "param_names": np.array(names)}
    with torch.no_grad():
        for key, ids in (("p", pids), ("q", qids), ("f", fids)):
            t = torch.from_numpy(ids).long()
            # the attention_mask argument is ignored by the reference: pass all ones
            e = ref.body_emb(t, torch.ones_like(t)).numpy()
            d = np.abs(orc.body_emb(t).numpy() - e).max()
            print(f"{key}: oracle vs reference max abs diff {d:.3g}")
            assert d < 2e-4
            out[key + "ids"], out[key + "emb"] = ids, e
        q, a, b = (torch.from_numpy(x).long() for x in (qids[:3], pids[:3], pids[3:]))
        loss = ref(q, torch.ones_like(q), a, torch.ones_like(a), b, torch.ones_like(b))[0]
        d = abs(float(orc.nll_loss(q, a, b)) - float(loss))
        print(f"loss {float(loss):.6f}: oracle diff {d:.3g}")
        assert d < 1e-4
    out["loss"] = np.float64(float(loss))
    path = os.path.join(GOLD, "encoder_seed.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


def golden_grads():
    rng = np.random.default_rng(1)
    vocab = 1000
    sd = random_seed_state_dict(seed=1, n_layer=2, vocab=vocab)
    ref = reference_seed_model(2, vocab, sd)
    q_ids = make_ids(rng, [32, 9, 20, 5], 32, vocab, holes=[(0, 11)])
    a_ids = make_ids(rng, [128, 70, 33, 100], 128, vocab, holes=[(1, 40)])
    b_ids = make_ids(rng, [90, 128, 64, 17], 128, vocab)
    q, a, b = (torch.from_numpy(x).long() for x in (q_ids, a_ids, b_ids))
    loss = ref(q, torch.ones_like(q), a, torch.ones_like(a), b, torch.ones_like(b))[0]
    loss.backward()
    grads = {n: p.grad for n, p in ref.named_parameters() if p.grad is not None}
    assert not any(n.startswith("classification_heads.") for n in grads)
    orc = SEEDDotOracle(sd, n_layer=2)
    leaves = orc.leaves()
    ol = orc.nll_loss(q, a, b)
    ol.backward()
    # the key biases' exact gradient is zero (softmax ignores a per-query constant): both sides hold rounding noise,
    # measured against the query bias's gradient instead
    worst = max(float((leaves[n].grad - g).norm() / grads[n.replace("k_proj", "q_proj")].norm())
                for n, g in grads.items())
    lv, olv = float(loss.detach()), float(ol.detach())
    print(f"grads: loss {lv:.6f} (oracle diff {abs(olv - lv):.3g}); worst relative gradient difference {worst:.3g}")
    assert worst < 1e-3
    names = list(grads)
    p = "seed_encoder.encoder.sentence_encoder."
    path = os.path.join(GOLD, "seed_grads.npz")
    np.savez_compressed(path, seed=np.int64(1), q_ids=q_ids, a_ids=a_ids, b_ids=b_ids, loss=np.float64(lv),
                        names=np.array(names), sketch=np.stack([grad_sketch(grads[n], n).numpy() for n in names]),
                        tok_pad_row=grads[p + "embed_tokens.weight"][PAD].numpy(),
                        pos_pad_row=grads[p + "embed_positions.weight"][PAD].numpy())
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    golden_grads()
    golden_embeddings()
