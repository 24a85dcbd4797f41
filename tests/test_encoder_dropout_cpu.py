"""Dropout of the trainable encoder, CPU side: the numpy Philox4x32-10 against Random123's known answers, the masks'
statistics and their independence of generation order, and the fp64 backward mirrors with masks against
torch.autograd, each perturbation of the backward's rules rejected."""
import numpy as np
import pytest
import torch

from tests import encoder_dropout_refs as D


@pytest.mark.parametrize("key, ctr, want", [
    ((0, 0), (0, 0, 0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF, 0xFFFFFFFF), (0xFFFFFFFF,) * 4, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0xA4093822, 0x299F31D0), (0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(key, ctr, want):
    assert tuple(int(x) for x in D.philox_key(*key, ctr)) == want


def test_dbg_bits_layout():
    """The test hook's counter: (lo, hi of first + i, lo, hi of stream_word), carrying into the high word."""
    seed, sw, first = 0x0123456789ABCDEF, 0xDEADBEEF00C0FFEE, 0xFFFFFFFE
    got = D.dbg_bits(seed, sw, first, 4).reshape(4, 4)
    for i in range(4):
        x = first + i
        ref = D.philox(seed, np.uint32(x & 0xFFFFFFFF), np.uint32(x >> 32), np.uint32(sw & 0xFFFFFFFF), np.uint32(sw >> 32))
        assert np.array_equal(got[i], ref)


def test_threshold_and_scale():
    for p in (0.1, 0.05, 0.3, 0.99):
        assert abs(D.p_eff(p) - p) <= 2 ** -17
    assert D.threshold(0.1) == 6554 and D.threshold(0.0) == 0 and D.threshold(0.9999999) == 65535
    assert D.scale(0.1) == float(np.float32(1) / np.float32(1 - 6554 / 65536))


def _sigma_ok(frac, n, p):
    q = 1 - D.p_eff(p)
    return abs(frac - q) <= 6 * np.sqrt(q * (1 - q) / n)


@pytest.mark.parametrize("p", [0.1, 0.3])
def test_keep_fraction_per_site(p):
    seed = 1234
    for site in (D.SITE_EMBED, D.SITE_ATTN_OUT, D.SITE_FFN_OUT):
        m = D.hidden_mask(seed, site, 3, np.arange(700), 768, p)
        assert _sigma_ok(m.mean(), m.size, p), (site, m.mean())
    a = D.attn_masks(seed, 2, 2, 3, 128, p)
    assert _sigma_ok(a.mean(), a.size, p)


def test_masks_of_different_sites_layers_heads_seeds_are_independent():
    """Two masks that share no counter agree where both keep at the independent rate q^2, and both drop at p^2."""
    p = 0.1
    q = 1 - D.p_eff(p)
    base = D.hidden_mask(7, D.SITE_ATTN_OUT, 1, np.arange(512), 768, p)
    others = {"site": D.hidden_mask(7, D.SITE_FFN_OUT, 1, np.arange(512), 768, p),
              "layer": D.hidden_mask(7, D.SITE_ATTN_OUT, 2, np.arange(512), 768, p),
              "seed": D.hidden_mask(8, D.SITE_ATTN_OUT, 1, np.arange(512), 768, p),
              "embedding site": D.hidden_mask(7, D.SITE_EMBED, 1, np.arange(512), 768, p)}
    n = base.size
    for name, o in others.items():
        both = (base * o).mean()
        assert abs(both - q * q) <= 6 * np.sqrt(q * q * (1 - q * q) / n), (name, both)
        assert not np.array_equal(base, o)
    a = D.attn_mask(7, 0, 1, 0, 12, 256, p)
    for name, o in {"head": D.attn_mask(7, 0, 1, 1, 12, 256, p), "sequence": D.attn_mask(7, 0, 2, 0, 12, 256, p),
                    "layer": D.attn_mask(7, 1, 1, 0, 12, 256, p), "seed": D.attn_mask(9, 0, 1, 0, 12, 256, p),
                    "transposed": a.T}.items():
        both = (a * o).mean()
        assert abs(both - q * q) <= 6 * np.sqrt(q * q * (1 - q * q) / a.size), (name, both)


def test_mask_is_independent_of_generation_order():
    """An element's decision depends on its logical index only: generating a permuted subset of tokens / queries gives
    the same rows."""
    rng = np.random.default_rng(0)
    full = D.hidden_mask(11, D.SITE_FFN_OUT, 4, np.arange(1024), 768, 0.1)
    perm = rng.permutation(1024)[:300]
    assert np.array_equal(D.hidden_mask(11, D.SITE_FFN_OUT, 4, perm, 768, 0.1), full[perm])
    fa = D.attn_mask(11, 3, 5, 7, 12, 512, 0.1)
    qs = rng.permutation(512)[:100]
    assert np.array_equal(D.attn_mask(11, 3, 5, 7, 12, 512, 0.1, queries=qs), fa[qs])
    # CLS rows of the pruned last layer: token r L of sequence r is the unpruned layer's row
    L = 256
    cls = D.hidden_mask(11, D.SITE_ATTN_OUT, 1, np.arange(4) * L, 768, 0.1)
    assert np.array_equal(cls, D.hidden_mask(11, D.SITE_ATTN_OUT, 1, np.arange(4 * L), 768, 0.1)[::L])


def _attn_inputs(L, seed):
    g = np.random.default_rng(seed)
    q, k, v = (g.standard_normal((L, 64)) for _ in range(3))
    kb = np.where(g.random(L) < 0.8, 0.0, -10000.0)
    kb[0] = 0.0
    do = g.standard_normal((L, 64))
    return q, k, v, kb, do


@pytest.mark.parametrize("L", [64, 256])
def test_attention_mirror_matches_autograd(L):
    q, k, v, kb, do = _attn_inputs(L, L)
    p = 0.1
    m = D.attn_mask(3, 0, 0, 0, 12, L, p)
    s = D.scale(p)
    tq, tk, tv = (torch.tensor(x, requires_grad=True) for x in (q, k, v))
    P = torch.softmax(tq @ tk.T / 8.0 + torch.tensor(kb)[None, :], dim=-1)
    ctx = (P * torch.tensor(m) * s) @ tv
    ctx.backward(torch.tensor(do))
    ref = [t.grad.numpy() for t in (tq, tk, tv)]
    got = D.attention_bwd(q, k, v, kb, do, m, s)
    ctx_mirror, _ = D.attention_fwd(q, k, v, kb, m, s)
    np.testing.assert_allclose(ctx_mirror, ctx.detach().numpy(), rtol=1e-10, atol=1e-12)
    for a, b in zip(got, ref):
        np.testing.assert_allclose(a, b, rtol=1e-9, atol=1e-11)
    # an fp32 emulation of the kernels' arithmetic stays within a bound the perturbations exceed
    f32 = [x.astype(np.float32).astype(np.float64) for x in (q, k, v, do)]
    emu = D.attention_bwd(f32[0], f32[1], f32[2], kb, f32[3], m, np.float32(s))
    bound = [1e-4 * (np.abs(r).max() + 1e-3) + 1e-5 for r in ref]
    for a, b, t in zip(emu, ref, bound):
        assert np.abs(a - b).max() <= t
    perts = {"mask not applied": dict(mask_bwd=False), "1/(1-p) missing": dict(scale_bwd=False),
             "D from the unmasked dO V^T": dict(d_from_unmasked=True), "mask indexed (j, i)": dict(transpose_mask=True)}
    for name, kw in perts.items():
        bad = D.attention_bwd(q, k, v, kb, do, m, s, **kw)
        assert max(np.abs(a - b).max() / t for a, b, t in zip(bad, ref, bound)) > 1.0, name


def test_hidden_site_mirror_matches_autograd():
    """T = m o (x W^T + b) s + R, then LayerNorm: the branch gets m o dT s (bias included), the residual dT."""
    g = np.random.default_rng(5)
    M, K, H = 48, 96, 256
    x, w, b, r = g.standard_normal((M, K)), g.standard_normal((H, K)) * 0.1, g.standard_normal(H), g.standard_normal((M, H))
    gam, dy = 1 + 0.1 * g.standard_normal(H), g.standard_normal((M, H))
    p = 0.1
    m = D.hidden_mask(2, D.SITE_ATTN_OUT, 0, np.arange(M), H, p)
    s = D.scale(p)
    tx, tw, tb, tr = (torch.tensor(a, requires_grad=True) for a in (x, w, b, r))
    T = (tx @ tw.T + tb) * torch.tensor(m) * s + tr
    y = torch.nn.functional.layer_norm(T, (H,), torch.tensor(gam), None, 1e-5)
    y.backward(torch.tensor(dy))
    dT, _, _ = D.layer_norm_bwd(T.detach().numpy(), gam, dy, 1e-5)
    dx, dw, db, dres = D.dropout_linear_bwd(dT, m, s, x, w)
    ref = (tx.grad.numpy(), tw.grad.numpy(), tb.grad.numpy(), tr.grad.numpy())
    for a, c in zip((dx, dw, db, dres), ref):
        np.testing.assert_allclose(a, c, rtol=1e-9, atol=1e-10)
    perts = {"mask not applied": dict(mask_bwd=False), "1/(1-p) missing": dict(scale_bwd=False),
             "residual gradient masked": dict(mask_residual=True), "bias gradient from the unmasked dT":
             dict(bias_unmasked=True)}
    for name, kw in perts.items():
        bad = D.dropout_linear_bwd(dT, m, s, x, w, **kw)
        rel = max(np.linalg.norm(a - c) / np.linalg.norm(c) for a, c in zip(bad, ref))
        assert rel > 0.03, name   # the end-to-end gate of the GPU tests is 0.03 / 0.05


def test_masked_attention_ref_matches_the_per_head_mirror():
    """The batched torch mirror the layer-by-layer GPU test uses against the per-head numpy one, every perturbation
    included, and against the unmasked reference at m = 1, s = 1."""
    from tests import encoder_grad_refs as G
    B, L, heads = 2, 64, 2
    H = heads * 64
    g = torch.Generator().manual_seed(3)
    qkv, do = torch.randn(B * L, 3 * H, generator=g, dtype=torch.float64), torch.randn(B * L, H, generator=g, dtype=torch.float64)
    kb = torch.where(torch.rand(B * L, generator=g) < 0.8, 0.0, -10000.0 * np.log2(np.e)).double()
    am = torch.tensor(D.attn_masks(5, 1, B, heads, L, 0.1))
    s = D.scale(0.1)
    flags = {None: {}, "no_mask_bwd": dict(mask_bwd=False), "no_scale_bwd": dict(scale_bwd=False),
             "d_unmasked": dict(d_from_unmasked=True), "mask_transposed": dict(transpose_mask=True)}
    for pert, kw in flags.items():
        ref = D.masked_attention_bwd_ref(qkv, kb, do, B, L, heads, am, s, pert).numpy()
        for b in range(B):
            for h in range(heads):
                rows = slice(b * L, (b + 1) * L)
                cols = [slice(c * H + h * 64, c * H + h * 64 + 64) for c in range(3)]
                q, k, v = (qkv[rows, c].numpy() for c in cols)
                mine = D.attention_bwd(q, k, v, kb[rows].numpy() / np.log2(np.e), do[rows, h * 64:h * 64 + 64].numpy(),
                                       am[b, h].numpy(), s, **kw)
                for x, c in zip(mine, cols):
                    np.testing.assert_allclose(ref[rows, c], x, rtol=1e-9, atol=1e-11)
    ones = torch.ones_like(am)
    np.testing.assert_allclose(D.masked_attention_bwd_ref(qkv, kb, do, B, L, heads, ones, 1.0).numpy(),
                               G.attention_bwd_ref(qkv, kb, do, B, L, heads).numpy(), rtol=1e-12, atol=1e-13)
