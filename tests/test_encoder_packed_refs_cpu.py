"""The fp64 mirror on a packed plan (no GPU needed): at exact arithmetic, the plan-aware mirror of encoder_layer_refs /
encoder_dropout_refs run on the packed rows of a batch gives the dense mirror's gradients of the same batch, every
parameter gradient and every row of d X_in gathered through row_tok, with and without dropout masks; and each packed
perturbation of the mirror changes some output on that data, so none of them is a no-op.  Plans come from the host-only
planner ance_dbg_pack_rows, the one ance_encoder_forward_train_packed uses."""
import ctypes as C

import numpy as np
import pytest
import torch

from ance_b200 import _lib
from tests import encoder_dropout_refs as D
from tests import encoder_layer_refs as LR
from tests.test_encoder_backward_cpu import _layer_weights, _tiny_model, _train_forward

F64 = torch.float64
HEADS, N_LAYER, P, SEED = 4, 2, 0.1, 0x5EED
PACKED_PERTURBATIONS = ("cls_residual_dense_rows", "wo_ctx_packed_rows", "attention_whole_tile", "position_from_row",
                        "hidden_mask_by_row", "attn_mask_from_tile")


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _plan(lib, lens, L, align):
    B = len(lens)
    lens = np.asarray(lens, np.int32)
    row0 = np.zeros(B, np.int32)
    tok = np.full(1 << 13, -7, np.int32)
    n_placed, n_tiles = C.c_int(), C.c_int()
    assert lib.ance_dbg_pack_rows(lens.ctypes.data, B, L, 1 << 13, align, row0.ctypes.data, tok.ctypes.data,
                                  C.byref(n_placed), C.byref(n_tiles)) == 0, lib.ance_last_error()
    assert n_placed.value == B
    M = n_tiles.value * 128
    return torch.from_numpy(row0).long(), torch.from_numpy(lens).long(), torch.from_numpy(tok[:M]).long(), M


def _batch(L, seed):
    """Prefix masks: lengths 1, L and a spread between (several short sequences share a tile)."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.tensor([L, 1, max(1, L - 3), max(1, L // 3), max(1, L // 8), 2, max(1, L // 2 + 1)])
    lens = torch.cat([lens, torch.randint(1, L + 1, (2,), generator=g)])
    B = len(lens)
    mask = torch.arange(L)[None, :] < lens[:, None]
    ids = torch.where(mask, torch.randint(3, 40, (B, L), generator=g), torch.ones(B, L, dtype=torch.long))
    ids[:, 0] = 0
    return ids, mask, lens


def _pack(x, tok, g):
    """Dense rows [B L, .] at their packed rows; rows of no sequence hold noise the mirror must never read into a sum."""
    out = torch.randn(len(tok), x.shape[1], generator=g, dtype=F64) * 3.0
    out[tok >= 0] = x[tok[tok >= 0]]
    return out


def _chains(sd, ids, mask, lens, plan, dropout, perturb=None, dense=True):
    """Head -> pruned last layer -> full layer -> embeddings, dense (unless dense=False) and on the plan, exact
    arithmetic.  -> [dense,] packed: {layer: grads}, the embedding grads under "emb" and d X_0 (dense rows) under "x0"."""
    B, L = ids.shape
    acts, kb, x_final, head_in, _ = _train_forward(sd, ids, mask, N_LAYER, HEADS, pad=1)
    d_out = torch.randn(B, 256, generator=torch.Generator().manual_seed(7), dtype=F64)
    gh, _ = LR.head_bwd_ref(d_out, head_in, x_final, sd["embeddingHead.weight"], sd["norm.weight"], exact=True)
    row0, _, tok, M = plan
    noise = torch.Generator().manual_seed(11)
    s = D.scale(P)
    out = []
    for packed in ((False, True) if dense else (True,)):
        dy, res = gh["x_final"], {}
        for l in reversed(range(N_LAYER)):
            last = l == N_LAYER - 1
            a = acts[l]
            if packed:
                a = {k: (_pack(v, tok, noise) if k in ("x_in", "qkv", "ctx") or not last else v) for k, v in a.items()}
                if last:
                    a["cls_ctx"] = acts[l]["ctx"][::L]
            kbias = torch.zeros(M, dtype=F64) if packed else kb   # the packed workspace's key bias is all zero
            w = _layer_weights(sd, l)
            pl = plan if packed else None
            pp = perturb if packed else None
            if dropout:
                if last:
                    hm = [torch.tensor(D.hidden_mask(SEED, site, l, np.arange(B) * L, 256, P)) for site in (2, 3)]
                elif packed:
                    hm = [torch.tensor(D.packed_hidden_mask(SEED, site, l, tok.numpy(), 256, P, pp)) for site in (2, 3)]
                else:
                    hm = [torch.tensor(D.hidden_mask(SEED, site, l, np.arange(B * L), 256, P)) for site in (2, 3)]
                am = torch.tensor(D.packed_attn_masks(SEED, l, B, HEADS, L, P, row0.numpy(), pp))
                g, _ = D.masked_layer_bwd_ref(a, kbias, w, dy, B, L, HEADS, last, 1e-5, "fp16", hm[0], hm[1], am, s,
                                              perturb=pp, plan=pl, exact=True)
            else:
                g, _ = LR.layer_bwd_ref(a, kbias, w, dy, B, L, HEADS, last, 1e-5, exact=True, perturb=pp, plan=pl)
            res[l] = g
            dy = g["x_in"]
        dx0 = LR.packed_to_dense(dy, tok, B * L) if packed else dy
        if dropout:
            m0 = D.packed_hidden_mask(SEED, 0, 0, tok.numpy(), 256, P, perturb if packed else None) if packed else \
                D.hidden_mask(SEED, 0, 0, np.arange(B * L), 256, P)
            if packed:
                m0 = LR.packed_to_dense(torch.tensor(m0), tok, B * L)
            dx0 = dx0 * torch.as_tensor(m0) * s
        shift = LR.position_from_row_shift(plan, lens, B, L) if (packed and perturb == "position_from_row") else 0
        e = lambda n: sd["roberta.embeddings." + n]
        res["emb"], _ = LR.embedding_stage_ref(ids, dx0, e("word_embeddings.weight"), e("position_embeddings.weight"),
                                               e("token_type_embeddings.weight"), e("LayerNorm.weight"), 1e-5, 1, True,
                                               pos_shift=shift)
        res["x0"] = dx0
        out.append(res)
    return out


def _flat(res, tok, B, L):
    """Every output of a chain as {name: dense tensor} (d X_in of the packed chain gathered to its dense tokens)."""
    f = {}
    for l in range(N_LAYER):
        for k, v in res[l].items():
            f[f"{l}.{k}"] = LR.packed_to_dense(v, tok, B * L) if (k == "x_in" and tok is not None) else v
    f.update({f"emb.{k}": v for k, v in res["emb"].items()})
    f["x0"] = res["x0"]
    return f


CASES = [(align, L) for align in (1, 16) for L in (16, 128, 256)]


@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("align,L", CASES)
def test_packed_mirror_equals_dense_mirror(lib, align, L, dropout):
    sd = _tiny_model(L, max_pos=L + 2)
    ids, mask, lens = _batch(L, L + align)
    B = len(lens)
    plan = _plan(lib, lens, L, align)
    tok = plan[2]
    dense, packed = _chains(sd, ids, mask, lens, plan, dropout)
    # rows of no sequence, and rows past a sequence's length, get exactly 0
    real = (tok >= 0) & ((tok % L) < lens[tok.clamp(min=0) // L])
    for l in range(N_LAYER):
        assert torch.count_nonzero(packed[l]["x_in"][~real]) == 0, l
    fd, fp = _flat(dense, None, B, L), _flat(packed, tok, B, L)
    assert set(fd) == set(fp)
    for k in fd:
        # the key bias's exact gradient is zero (softmax is shift-invariant per query): fp64 noise on both sides
        scale = float(fd[k.replace("k_b", "q_b") if k.endswith(".k_b") else k].abs().max())
        assert torch.allclose(fp[k], fd[k], rtol=1e-10, atol=1e-12 * scale), (k, float((fp[k] - fd[k]).abs().max()), scale)


@pytest.mark.parametrize("align,L", CASES)
def test_every_packed_perturbation_changes_the_mirror(lib, align, L):
    """Each packed perturbation moves some output well past fp64 noise on a plan where it applies: the whole-tile
    attention needs L <= 128, the dropout masks the dropout chain; the attention masks from the tile need align 16 (the
    packed forward refuses attention dropout on align 1); the CLS residual at rows b L and the masks keyed by row need a
    plan whose rows are not the dense tokens themselves."""
    sd = _tiny_model(L, max_pos=L + 2)
    ids, mask, lens = _batch(L, L + align)
    B = len(lens)
    plan = _plan(lib, lens, L, align)
    assert bool((plan[0] % 128 != 0).any()), "a sequence placed inside a tile"
    rows = torch.nonzero(plan[2] >= 0).flatten()
    identity = torch.equal(plan[2][rows], rows)
    base = {d: _flat(_chains(sd, ids, mask, lens, plan, d, dense=False)[0], plan[2], B, L) for d in (False, True)}
    for pn in PACKED_PERTURBATIONS:
        if pn == "attention_whole_tile" and L > 128:
            continue
        if pn == "attn_mask_from_tile" and align != 16:
            continue
        if pn in ("cls_residual_dense_rows", "hidden_mask_by_row") and identity:
            continue   # align 16, L = 16: row b L + i is token b L + i already

        dropout = pn in ("hidden_mask_by_row", "attn_mask_from_tile")
        pert = _flat(_chains(sd, ids, mask, lens, plan, dropout, perturb=pn, dense=False)[0], plan[2], B, L)
        moved = max(float((pert[k] - base[dropout][k]).abs().max() / base[dropout][k].abs().max().clamp_min(1e-300))
                    for k in pert)
        assert moved > 1e-6, (pn, moved)
