"""CPU half of the encoder kernel tests: the error models of tests/encoder_refs.py against fp32 emulations of the kernels'
arithmetic (correct arithmetic inside, every perturbed reference outside), the GELU coefficients of gemm_store.cuh within
their documented bounds, the references tied to the fp32 oracle, and the test hooks' argument checks without a GPU."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
from scipy.special import erf as sp_erf

from tests import encoder_refs as R

GEN_SEED = 20261016


def _gelu64(x):
    x = np.asarray(x, dtype=np.float64)
    return 0.5 * x * (1.0 + sp_erf(x / math.sqrt(2.0)))


def _gelu_grid():
    f = np.float32
    lin = np.linspace(-40.0, 40.0, 4_000_001, dtype=np.float64)
    lg = np.logspace(-8, 4, 200_001)
    return np.unique(np.concatenate([lin, lg, -lg, [0.0]]).astype(f))


@pytest.mark.parametrize("act,measured", [(1, 7.07e-7), (2, 3.63e-6)])
def test_gelu_forms_within_documented_bounds(act, measured):
    """Both GELU forms of the epilogue, emulated in fp32 from the coefficients parsed out of gemm_store.cuh, against
    erf-GELU in fp64 over |x| <= 1e4: max error within the documented bound (DESIGN.md 4.1: 7.1e-7 erfc form, 3.7e-6
    logistic form) and not far below it (an edited coefficient moves it); exact saturation out to +-1e30."""
    erf_c, log_c = R.gelu_coefficients()
    assert len(erf_c) == 10 and len(log_c) == 7, (erf_c, log_c)
    emu = (lambda x: R.gelu_erf2_emulate(x, erf_c)) if act == 1 else (lambda x: R.gelu_logistic2_emulate(x, log_c))
    x = _gelu_grid()
    err = np.abs(emu(x).astype(np.float64) - _gelu64(x))
    worst = float(err.max())
    print(f"GELU act {act}: max |err| {worst:.3e} at x = {x[err.argmax()]:.4f} (bound {R.GELU_BOUND[act]:.1e})")
    assert worst <= R.GELU_BOUND[act], worst
    assert worst >= 0.9 * measured, worst
    big = np.array([1e5, 1e10, 1e30, -1e5, -1e10, -1e30, 65504.0, -65504.0], dtype=np.float32)
    y = emu(big)
    assert np.all(np.isfinite(y))
    assert np.array_equal(y[big > 0], big[big > 0]) and np.all(y[big < 0] == 0.0)
    # the tanh approximation lies well outside either bound: a kernel computing it cannot pass the GELU sweep
    xt = torch.from_numpy(x.astype(np.float64))
    assert (R.gelu_tanh(xt) - R.gelu_erf(xt)).abs().max().item() > 50 * R.GELU_BOUND[2]
    # the fp64 reference GELU used by the GPU tests is scipy's erf-GELU
    assert np.abs(R.gelu_erf(xt).numpy() - _gelu64(x)).max() <= 1e-12


def _emulate_linear(A, W, bias, Rs, act, fmt):
    """linear<FMT> in fp32: fp32 accumulation, + bias, GELU form `act`, + residual, 16-bit output."""
    x = (A.float() @ W.float().T)
    if bias is not None:
        x = x + bias.float()
    if act:
        erf_c, log_c = R.gelu_coefficients()
        xn = x.numpy()
        x = torch.from_numpy(R.gelu_erf2_emulate(xn, erf_c) if act == 1 else R.gelu_logistic2_emulate(xn, log_c))
    if Rs is not None:
        x = x + Rs.float()
    return x.to(R.dtype16(fmt)).to(torch.float64)


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_linear_error_model_against_emulation(fmt, act):
    g = torch.Generator().manual_seed(GEN_SEED + act)
    M, N, K = 96, 256, 768
    A = R.round16(torch.randn(M, K, generator=g, dtype=torch.float64), fmt)
    W = R.round16(torch.randn(N, K, generator=g, dtype=torch.float64) * 0.04, fmt)
    bias = torch.randn(N, generator=g, dtype=torch.float64).float().double()
    Rs = R.round16(torch.randn(M, N, generator=g, dtype=torch.float64), fmt)
    out = _emulate_linear(A, W, bias, Rs, act, fmt)
    x, y = R.linear_ref(A, W, bias, Rs, act)
    tol = R.linear_tol(A, W, x, y, Rs, act, fmt)
    pert = {"bias n+1": R.linear_ref(A, W, bias, Rs, act, bias_shift=1)[1],
            "residual row+1": R.linear_ref(A, W, bias, Rs, act, res_shift=1)[1]}
    err, rep = R.discrimination(out, y, tol, pert)
    print(f"linear {fmt} act {act}: max err/tol {err:.3f}, perturbed {rep}")
    assert err <= 1.0
    for name, (frac, margin, rows) in rep.items():
        assert rows >= M // 2 and frac == 1.0, (name, rep)


def _attention_case(fmt, L, B, heads, seed):
    """Dense qkv with prefix masks and planted peaks in blocks 1..3 (only rows 5 and 17 of each 32-row warp planted)."""
    g = torch.Generator().manual_seed(seed)
    n = B * L
    qkv = R.random_qkv(n, heads, fmt, g)
    lens = [L, L - 33, 129 if L > 129 else L // 2 + 1, 1][:B]
    keep = torch.zeros(n, dtype=torch.bool)
    for b, ln in enumerate(lens):
        keep[b * L:b * L + ln] = True
    deltas = [4.0, 7.9, 8.1, 12.0, 30.0, 120.0, 200.0]
    planted, slot = [], {}
    k = 0
    for b, ln in enumerate(lens):
        if ln <= 128:
            continue
        for j in range(1, (ln - 1) // 128 + 1):
            for r in (5, 17, 37 + 32 * j):
                row = b * L + r
                if r >= ln:
                    continue
                head = k % heads
                key = b * L + min(j * 128 + (k * 37) % 128, ln - 1)
                s = slot.get((b, head), 0)
                slot[(b, head)] = s + 1
                d = R.plant(qkv, heads, fmt, row, head, key, list(range(b * L, b * L + j * 128)), deltas[k % len(deltas)], s)
                planted.append((row, head, j, d))
                k += 1
    # the reverse: a huge maximum in block 0, far lower later blocks
    if lens[0] > 128:
        s = slot.get((0, 0), 0)
        R.plant(qkv, heads, fmt, 70, 0, 3, [i for i in range(lens[0]) if i != 3], 200.0, s)
    lo = torch.arange(n) // L * L
    return qkv, keep, lo, lo + L, planted


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
@pytest.mark.parametrize("L,B", [(512, 2), (256, 3), (128, 2), (64, 3)])
def test_attention_error_model_against_emulation(fmt, L, B):
    """attention_emulate (the kernel's fp32 block arithmetic with the > 8 log2-unit redo voted per 32-row warp) lies
    within attention_ref's tolerance; the three perturbed references (key range one further, no alpha rescale, last real
    key masked) lie outside it."""
    heads = 2
    qkv, keep, lo, hi, planted = _attention_case(fmt, L, B, heads, GEN_SEED + L)
    out = R.attention_emulate(qkv, heads, L, keep, fmt)
    ref, tol = R.attention_ref(qkv, heads, lo, hi, keep, fmt)
    lens = keep.view(B, L).sum(1)
    k_ext = keep.clone().view(B, L)
    k_cut = keep.clone().view(B, L)
    for b in range(B):
        if lens[b] < L:
            k_ext[b, lens[b]] = True
        if lens[b] >= 2:
            k_cut[b, lens[b] - 1] = False
    pert = {"key range +1": R.attention_ref(qkv, heads, lo, hi, k_ext.flatten(), fmt)[0],
            "last key masked": R.attention_ref(qkv, heads, lo, hi, k_cut.flatten(), fmt)[0]}
    if L > 128:
        pert["no alpha rescale"] = R.attention_no_rescale_ref(qkv, heads, L, keep)
    err, rep = R.discrimination(out, ref, tol, pert)
    print(f"attention emulation {fmt} L {L}: max err/tol {err:.3f}, planted {len(planted)}, perturbed {rep}")
    assert err <= 1.0
    assert rep["last key masked"][2] >= B - 1 and rep["last key masked"][0] == 1.0, rep
    if any(ln < L for ln in lens.tolist()):
        assert rep["key range +1"][2] >= 1 and rep["key range +1"][0] == 1.0, rep
    if L > 128:
        assert any(d > 8.0 for *_, d in planted) and any(d < 8.0 for *_, d in planted)
        assert rep["no alpha rescale"][2] >= 1 and rep["no alpha rescale"][0] == 1.0, rep


@pytest.mark.parametrize("fmt", ["fp16", "bf16", None])
def test_layer_norm_error_model_against_emulation(fmt):
    """A plain fp32 LayerNorm (torch, CPU) lies within layer_norm_tol; unbiased variance and eps outside the square root
    lie outside it (rows of small variance, where eps matters)."""
    g = torch.Generator().manual_seed(GEN_SEED + 7)
    H = 768
    x = torch.randn(64, H, generator=g, dtype=torch.float64) * 0.05
    x[32:] += 1e3
    x = x.float().double() if fmt is None else R.round16(x[:32], fmt)
    gam = (1.0 + 0.05 * torch.randn(H, generator=g, dtype=torch.float64)).float().double()
    bet = (0.05 * torch.randn(H, generator=g, dtype=torch.float64)).float().double()
    eps = 1e-5
    y32 = torch.nn.functional.layer_norm(x.float(), (H,), gam.float(), bet.float(), eps).double()
    out = y32 if fmt is None else R.round16(y32, fmt)
    y, z = R.layer_norm_ref(x, gam, bet, eps)
    tol = R.layer_norm_tol(x, z, y, gam, bet, fmt)
    pert = {"unbiased var": R.layer_norm_ref(x, gam, bet, eps, unbiased=True)[0],
            "eps outside sqrt": R.layer_norm_ref(x, gam, bet, eps, eps_outside=True)[0]}
    err, rep = R.discrimination(out, y, tol, pert, changed_rows=torch.arange(x.shape[0]) < 32)
    print(f"layer norm {fmt}: max err/tol {err:.3f}, perturbed {rep}")
    assert err <= 1.0
    if fmt is None or fmt == "fp16":
        for name, (frac, margin, rows) in rep.items():
            assert rows >= 16 and frac == 1.0, (name, rep)


def test_refs_tied_to_fp32_oracle():
    """embed_ref, linear_ref, attention_ref and layer_norm_ref chained into one RoBERTa layer reproduce
    oracle/encoder_oracle.py's hidden states up to fp32 rounding."""
    from oracle.encoder_oracle import EncoderOracle, random_roberta_state_dict
    sd = random_roberta_state_dict(seed=5, n_layer=1, hidden=256, ffn=1024, vocab=1000, max_pos=80, head=False)
    orc = EncoderOracle(sd, "roberta.", "roberta", 1, 4, 1, 1e-5)
    g = torch.Generator().manual_seed(1)
    B, L = 3, 64
    ids = torch.randint(3, 1000, (B, L), generator=g)
    lens = torch.tensor([64, 20, 1])
    mask = torch.arange(L)[None, :] < lens[:, None]
    ids[~mask] = 1
    hs = orc.hidden_states(ids, mask)
    w = {k[len("roberta."):]: v.double() for k, v in sd.items()}
    x32, y0, _ = R.embed_ref(ids, w["embeddings.word_embeddings.weight"], w["embeddings.position_embeddings.weight"],
                             w["embeddings.token_type_embeddings.weight"], w["embeddings.LayerNorm.weight"],
                             w["embeddings.LayerNorm.bias"], 1e-5, True, 1)
    assert (y0 - hs[0].double()).abs().max().item() <= 1e-5
    X = y0.reshape(B * L, -1)
    p = "encoder.layer.0."
    Wqkv = torch.cat([w[p + f"attention.self.{n}.weight"] for n in ("query", "key", "value")])
    bqkv = torch.cat([w[p + f"attention.self.{n}.bias"] for n in ("query", "key", "value")])
    _, qkv = R.linear_ref(X, Wqkv, bqkv)
    lo = torch.arange(B * L) // L * L
    ctx, _ = R.attention_ref(qkv, 4, lo, lo + L, mask.flatten())
    _, t = R.linear_ref(ctx, w[p + "attention.output.dense.weight"], w[p + "attention.output.dense.bias"], X)
    x1, _ = R.layer_norm_ref(t, w[p + "attention.output.LayerNorm.weight"], w[p + "attention.output.LayerNorm.bias"], 1e-5)
    _, f = R.linear_ref(x1, w[p + "intermediate.dense.weight"], w[p + "intermediate.dense.bias"], act=2)
    _, t2 = R.linear_ref(f, w[p + "output.dense.weight"], w[p + "output.dense.bias"], x1)
    x2, _ = R.layer_norm_ref(t2, w[p + "output.LayerNorm.weight"], w[p + "output.LayerNorm.bias"], 1e-5)
    d = (x2.reshape(B, L, -1) - hs[1].double()).abs()
    assert d.max().item() <= 1e-4, d.max().item()


_FAKE = 1 << 20   # a 16-byte-aligned address that is never dereferenced: every call below stops before any device work


def test_kernel_hooks_refuse_without_gpu(lib):
    """The three kernel hooks: ANCE_ERR_INVALID (1) for bad shapes before anything else, ANCE_ERR_CUDA (2) for valid
    shapes without an sm_90 device."""
    p = _FAKE
    assert lib.ance_dbg_linear(0, p, 760, 128, p, 768, 768, p, None, 0, 0, p, None, None) == 1        # lda < K
    assert lib.ance_dbg_linear(0, p, 768, 128, p, 768, 768, p, p, 764, 0, p, None, None) == 1        # ldr < N
    assert lib.ance_dbg_linear(0, p, 768, 128, p, 768, 768, p, None, 0, 3, p, None, None) == 1        # act 3
    assert lib.ance_dbg_linear(0, p, 768, 128, p, 768, 768, p, None, 0, 0, None, None, None) == 1     # no output
    assert lib.ance_dbg_linear(0, p + 2, 768, 128, p, 768, 768, p, None, 0, 0, p, None, None) == 1    # misaligned
    assert lib.ance_dbg_linear(5, p, 768, 128, p, 768, 768, p, None, 0, 0, p, None, None) == 1        # format
    assert lib.ance_dbg_attention(0, p, 384, 100, 12, p, None, None, None, p, None) == 1   # L neither /128 nor | 128
    assert lib.ance_dbg_attention(0, p, 300, 128, 12, p, None, None, None, p, None) == 1   # n_tokens % L
    assert lib.ance_dbg_attention(0, p, 300, 256, 12, p, p, p, p, p, None) == 1            # plan: n_tokens % 128
    assert lib.ance_dbg_attention(0, p, 384, 256, 12, p, p, p, None, p, None) == 1         # L > 128 without tile_kv
    assert lib.ance_dbg_attention(0, p, 384, 64, 12, p, p, p, p, p, None) == 1             # tile_kv at L <= 128
    assert lib.ance_dbg_attention(0, p, 384, 128, 17, p, None, None, None, p, None) == 1   # heads
    assert lib.ance_dbg_layer_norm(0, p, 0, 768, 10, 640, p, p, 1e-5, p, None, 2, None) == 1   # H
    assert lib.ance_dbg_layer_norm(0, p, 0, 700, 10, 768, p, p, 1e-5, p, None, 2, None) == 1   # in_ld
    assert lib.ance_dbg_layer_norm(0, p, 0, 768, 10, 768, p, p, 1e-5, p, None, 5, None) == 1   # rows_per_warp
    assert lib.ance_dbg_layer_norm(0, p, 0, 768, 10, 768, p, p, 1e-5, None, None, 2, None) == 1
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device errors are not reachable")
    assert lib.ance_dbg_linear(0, p, 768, 128, p, 768, 768, p, p, 768, 2, p, None, None) == 2
    assert lib.ance_dbg_linear(1, p, 2304, 5, p, 768, 768, None, p, 98304, 0, None, p, None) == 2
    assert lib.ance_dbg_attention(0, p, 1024, 512, 12, p, None, None, None, p, None) == 2
    assert lib.ance_dbg_attention(1, p, 1024, 256, 12, p, p, p, p, p, None) == 2
    assert lib.ance_dbg_layer_norm(0, p, 1, 768, 10, 768, p, p, 1e-5, None, p, 4, None) == 2


def test_linear_discrimination_blocked_matches_whole_matrix():
    """The row-blocked fp64 check of the wide-tile tests gives the whole-matrix discrimination() result (bias n+1 and
    residual row+1 through linear_ref's own perturbations), and each of its tile-layout perturbations, played back (in
    fp64) as a kernel output, is caught: out of bound against the reference and within bound of its own perturbed
    reference."""
    g = torch.Generator().manual_seed(GEN_SEED + 7)
    M, N, K, fmt = 700, 776, 64, "bf16"
    A = R.round16(torch.randn(M, K, generator=g, dtype=torch.float64), fmt)
    W = R.round16(torch.randn(N, K, generator=g, dtype=torch.float64) * 0.04, fmt)
    b = torch.randn(N, generator=g).double()
    Rs = R.round16(torch.randn(M, N, generator=g, dtype=torch.float64), fmt)
    x, y = R.linear_ref(A, W, b, Rs)
    tol = R.linear_tol(A, W, x, y, Rs, 0, fmt)
    out = R.round16(y, fmt)
    whole = R.discrimination(out, y, tol, {"bias n+1": R.linear_ref(A, W, b, Rs, bias_shift=1)[1],
                                           "residual row+1": R.linear_ref(A, W, b, Rs, res_shift=1)[1]})
    err, rep = R.linear_discrimination_blocked(out, A, W, b, Rs, fmt, block_elems=256 * N)   # 3 blocks, the last ragged
    assert err == pytest.approx(whole[0], rel=1e-12) and err <= 1.0
    assert set(rep) == set(R.LINEAR_WIDE_PERTURBATIONS)
    for k in whole[1]:
        assert rep[k][0] == whole[1][k][0] == 1.0 and rep[k][2] == whole[1][k][2], (k, rep[k], whole[1][k])
        assert rep[k][1] == pytest.approx(whole[1][k][1], rel=1e-12)
    rows, cols = torch.arange(M), torch.arange(N)
    acc = A @ W.T
    bugs = {"bias n+1": acc + torch.roll(b, -1) + Rs, "residual row+1": acc + b + Rs[(rows + 1) % M],
            "residual row^64": acc + b + Rs[torch.where((rows ^ 64) < M, rows ^ 64, rows)],
            "acc col^64": acc[:, torch.where((cols ^ 64) < N, cols ^ 64, cols)] + b + Rs,
            "acc row^8": acc[torch.where((rows ^ 8) < M, rows ^ 8, rows)] + b + Rs}
    for name, bad in bugs.items():
        e, r = R.linear_discrimination_blocked(bad, A, W, b, Rs, fmt, block_elems=256 * N)
        assert e > 1.0 and r[name][0] == 0.0 and r[name][2] >= M // 2, (name, e, r[name])
    # without bias and residual only the accumulator perturbations apply
    _, r = R.linear_discrimination_blocked(R.round16(acc, fmt), A, W, None, None, fmt)
    assert set(r) == {"acc col^64", "acc row^8"} and all(v[0] == 1.0 for v in r.values())
