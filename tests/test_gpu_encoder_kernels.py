"""Encoder kernels one at a time against the fp64 references of tests/encoder_refs.py, through the hooks that launch the
encoder's own instantiations (ance_dbg_linear / ance_dbg_attention / ance_dbg_layer_norm, ance_encoder_debug_hidden).

Each family is held to the per-element tolerance of its written error model (encoder_refs.py docstrings), in fp16 and
bf16, and every test also shows that the tolerance discriminates: perturbed references (the outputs of plausible kernel
bugs) must lie outside it.  Output buffers carry guard rows filled with a sentinel bit pattern that must survive.  Each
test prints its measured maximum error as a fraction of the bound and the median margin by which each perturbed
reference was rejected."""
import ctypes as C

import numpy as np
import pytest
import torch

from ance_b200 import _lib
from tests import encoder_refs as R

pytestmark = pytest.mark.gpu

FMTS = ["fp16", "bf16"]
FMT_CODE = {"fp16": _lib.ANCE_FMT_FP16, "bf16": _lib.ANCE_FMT_BF16}
GUARD = 64                      # guard rows before and after every output
SENT16 = 0x7E5A                 # a NaN in fp16 and in bf16
SENT32 = 0x7FC0DEAD             # a NaN in fp32
F64 = torch.float64


@pytest.fixture(scope="module")
def gpu_lib():
    assert torch.cuda.is_available()
    return _lib.load()


def _st():
    return _lib.current_stream()


def _t16(x64, fmt):
    return x64.to(R.dtype16(fmt)).contiguous()


def _guarded(rows, cols, kind):
    """(flat buffer, [rows, cols] view inside it) with GUARD sentinel rows on either side."""
    n = (rows + 2 * GUARD) * cols
    if kind == "f32":
        buf = torch.full((n,), SENT32, dtype=torch.int32, device="cuda").view(torch.float32)
    else:
        buf = torch.full((n,), SENT16, dtype=torch.int16, device="cuda").view(R.dtype16(kind))
    return buf, buf[GUARD * cols:(GUARD + rows) * cols].view(rows, cols)


def _guards_intact(buf, rows, cols):
    raw = buf.view(torch.int32) if buf.dtype == torch.float32 else buf.view(torch.int16)
    want = SENT32 if buf.dtype == torch.float32 else SENT16
    head, tail = raw[:GUARD * cols], raw[(GUARD + rows) * cols:]
    assert bool((head == want).all()) and bool((tail == want).all()), "a guard row was overwritten"


def _check(name, out, ref, tol, pert, changed_rows=None, min_rows=1):
    err, rep = R.discrimination(out, ref, tol, pert, changed_rows)
    print(f"{name}: max err / bound {err:.3f}; perturbed (fraction rejected, median margin, rows) {rep}")
    assert err <= 1.0, f"{name}: max err / bound {err}"
    for k, (frac, margin, rows) in rep.items():
        assert rows >= min_rows and (rows == 0 or frac == 1.0), (name, k, rep)
    return err, rep


# ------------------------------------------------------------------------------------------------
# linear<FMT>
# ------------------------------------------------------------------------------------------------
def _linear_operands(M, N, K, fmt, seed, lda=None, ldr=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lda, ldr = lda or K, ldr or N
    Abuf = _t16(torch.randn((M - 1) * lda + K, generator=g, device="cuda", dtype=F64), fmt)
    A = Abuf.as_strided((M, K), (lda, 1))
    W = _t16(torch.randn(N, K, generator=g, device="cuda", dtype=F64) * 0.04, fmt)
    bias = torch.randn(N, generator=g, device="cuda", dtype=torch.float32)
    Rbuf = _t16(torch.randn((M - 1) * ldr + N, generator=g, device="cuda", dtype=F64), fmt)
    Rv = Rbuf.as_strided((M, N), (ldr, 1))
    return Abuf, A, W, bias, Rbuf, Rv


def _run_linear(gpu_lib, fmt, Abuf, lda, M, W, N, K, bias, Rbuf, ldr, act, out):
    """out: 'c16' or 'c32'.  Returns the output as fp64 [M, N] after checking its guards."""
    kind = fmt if out == "c16" else "f32"
    buf, view = _guarded(M, N, kind)
    rc = gpu_lib.ance_dbg_linear(FMT_CODE[fmt], Abuf.data_ptr(), lda, M, W.data_ptr(), N, K,
                            None if bias is None else bias.data_ptr(), None if Rbuf is None else Rbuf.data_ptr(),
                            ldr if Rbuf is not None else 0, act, view.data_ptr() if out == "c16" else None,
                            view.data_ptr() if out == "c32" else None, _st())
    assert rc == 0, gpu_lib.ance_last_error()
    torch.cuda.synchronize()
    _guards_intact(buf, M, N)
    return view.to(F64)


def _linear_case(gpu_lib, fmt, M, N, K, bias_on, act, res_on, out, seed, lda=None, ldr=None):
    lda_, ldr_ = lda or K, ldr or N
    Abuf, A, W, bias, Rbuf, Rv = _linear_operands(M, N, K, fmt, seed, lda_, ldr_)
    b = bias if bias_on else None
    rb, rv = (Rbuf, Rv) if res_on else (None, None)
    got = _run_linear(gpu_lib, fmt, Abuf, lda_, M, W, N, K, b, rb, ldr_, act, out)
    x, y = R.linear_ref(A, W, b, rv, act)
    tol = R.linear_tol(A, W, x, y, rv, act, fmt if out == "c16" else None)
    pert = {}
    if bias_on and N > 1:
        pert["bias n+1"] = R.linear_ref(A, W, b, rv, act, bias_shift=1)[1]
    if res_on and M > 1:
        pert["residual row+1"] = R.linear_ref(A, W, b, rv, act, res_shift=1)[1]
    return _check(f"linear {fmt} M{M} N{N} K{K} bias{int(bias_on)} act{act} res{int(res_on)} {out} lda{lda_} ldr{ldr_}",
                  got, y, tol, pert, min_rows=max(1, M // 2))


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("NK", [(768, 768), (2304, 768), (3072, 768), (768, 3072), (3072, 3072), (256, 256), (1024, 1024)])
def test_linear_shapes(gpu_lib, fmt, NK):
    N, K = NK
    for i, M in enumerate((1, 5, 127, 128, 129, 1000, 4097)):
        _linear_case(gpu_lib, fmt, M, N, K, True, (0, 2, 1)[i % 3], True, "c16", seed=M * 7 + N + K)
        _linear_case(gpu_lib, fmt, M, N, K, True, 2, False, "c32", seed=M * 11 + N + K)


@pytest.mark.parametrize("fmt", FMTS)
def test_linear_epilogue_combinations(gpu_lib, fmt):
    """Every combination of bias, act 0 / 1 / 2, residual and 16-bit vs fp32 output, dense and with the pruned last
    layer's strided views (A and residual rows at pitch L*H, M = B rows)."""
    for bias_on in (False, True):
        for act in (0, 1, 2):
            for res_on in (False, True):
                for out in ("c16", "c32"):
                    _linear_case(gpu_lib, fmt, 129, 768, 768, bias_on, act, res_on, out, seed=act * 4 + res_on * 2 + bias_on)
                    _linear_case(gpu_lib, fmt, 37, 768, 768, bias_on, act, res_on, out, seed=99 + act, lda=128 * 768, ldr=128 * 768)
    _linear_case(gpu_lib, fmt, 21, 768, 3072, True, 0, True, "c16", seed=5, lda=512 * 3072, ldr=512 * 768)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("act", [1, 2])
def test_linear_gelu_sweep(gpu_lib, fmt, act):
    """Exact chosen x in the accumulator (one-hot A rows times a 16-bit B column, plus an fp32 bias): the GELU of the
    epilogue over [-40, 40], tiny / subnormal / near-zero arguments and +-65504, fp32 output, against erf-GELU in fp64
    with the act-1 / act-2 bounds; the tanh-approximate GELU must be rejected."""
    K, N = 64, 1024
    M = K
    special = torch.tensor([65504.0, -65504.0, 6e-8, -6e-8, 1e-7, -1e-7, 1e-5, -1e-5, 1e-3, -1e-3, 0.0, 5e-3, -5e-3, 0.1,
                            -0.1, 0.5, -0.5, 1.0, -1.0, 2.0, -2.0, 3.0, -3.0, 6.0, -6.0, 9.0, -9.0, 20.0, -20.0, 30.0, -30.0,
                            40.0], dtype=F64)   # column 0 of B: added to a zero bias, so x is exactly these values
    xs = torch.cat([special, torch.linspace(-40, 40, N * K - 64, dtype=F64)])
    xs = torch.cat([xs, torch.zeros(N * K - xs.numel(), dtype=F64)]).view(N, K).cuda()
    Wv = R.round16(xs, fmt)
    g = torch.Generator(device="cuda").manual_seed(act)
    bias = (torch.randn(N, generator=g, device="cuda", dtype=torch.float32) * 1e-3)
    bias[:4] = 0.0
    A = torch.zeros(M, K, dtype=F64, device="cuda")
    A[torch.arange(M), torch.arange(M) % K] = 1.0
    A16, W16 = _t16(A, fmt), _t16(Wv, fmt)
    got = _run_linear(gpu_lib, fmt, A16, K, M, W16, N, K, bias, None, 0, act, "c32")
    x, y = R.linear_ref(A, Wv, bias.double(), None, act)
    tol = R.linear_tol(A, Wv, x, y, None, act, None)
    assert (x.abs() >= 40).any() and (x.abs() < 1e-6).any()
    pert = {"tanh GELU": R.linear_ref(A, Wv, bias.double(), None, act, gelu=R.gelu_tanh)[1]}
    _check(f"GELU sweep {fmt} act {act}", got, y, tol, pert, min_rows=M // 2)


@pytest.mark.parametrize("fmt", FMTS)
def test_dbg_gemm_variants(gpu_lib, fmt):
    """The five ance_dbg_gemm tilings (bf16 output and residual) at the bring-up shapes of tools/bringup_gemm.py."""
    for variant in range(5):
        for i, (M, N, K) in enumerate(((256, 512, 128), (1000, 776, 768), (8192, 3072, 768), (8192, 768, 3072))):
            Abuf, A, W, bias, Rbuf, Rv = _linear_operands(M, N, K, fmt, seed=variant * 13 + M)
            Rb = Rv.to(torch.bfloat16).contiguous()
            for act in ((variant + i) % 3,):
                buf, view = _guarded(M, N, "bf16")
                rc = gpu_lib.ance_dbg_gemm(Abuf.data_ptr(), W.data_ptr(), M, N, K, FMT_CODE[fmt], variant, bias.data_ptr(),
                                      Rb.data_ptr(), act, view.data_ptr(), None, _st())
                assert rc == 0, gpu_lib.ance_last_error()
                torch.cuda.synchronize()
                _guards_intact(buf, M, N)
                x, y = R.linear_ref(A, W, bias, Rb, act)
                tol = R.linear_tol(A, W, x, y, Rb, act, "bf16")
                _check(f"ance_dbg_gemm {fmt} variant {variant} M{M} N{N} K{K} act {act}", view.to(F64), y, tol,
                       {"bias n+1": R.linear_ref(A, W, bias, Rb, act, bias_shift=1)[1]}, min_rows=M // 2)


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def _run_attention(gpu_lib, fmt, qkv16, n, L, heads, kbias, lo=None, hi=None, tile_kv=None):
    H = heads * 64
    buf, view = _guarded(n, H, fmt)
    rc = gpu_lib.ance_dbg_attention(FMT_CODE[fmt], qkv16.data_ptr(), n, L, heads, kbias.data_ptr(),
                               None if lo is None else lo.data_ptr(), None if hi is None else hi.data_ptr(),
                               None if tile_kv is None else tile_kv.data_ptr(), view.data_ptr(), _st())
    assert rc == 0, gpu_lib.ance_last_error()
    torch.cuda.synchronize()
    _guards_intact(buf, n, H)
    return view.to(F64)


def _plant_dense(qkv, heads, fmt, L, lens, seq0):
    """Peaked rows in blocks 1..3: rows 5 and 17 of the first warp and one row of a later warp planted, every other row of
    those warps left flat (the per-warp redo vote is split), plus the reverse (a huge maximum in block 0)."""
    deltas = [4.0, 7.9, 8.1, 12.0, 30.0, 120.0, 200.0]
    planted, slot, k = [], {}, 0
    for b, ln in enumerate(lens):
        if ln <= 128:
            continue
        base = seq0 + b * L
        for j in range(1, (ln - 1) // 128 + 1):
            for r in (5, 17, 37 + 32 * j):
                if r >= ln:
                    continue
                head = k % heads
                s = slot.get((b, head), 0)
                if s >= len(R.PLANT_COORDS):
                    continue
                slot[(b, head)] = s + 1
                key = base + min(j * 128 + (k * 37) % 128, ln - 1)
                d = R.plant(qkv, heads, fmt, base + r, head, key, list(range(base, base + j * 128)), deltas[k % 7], s)
                planted.append(d)
                k += 1
        head = 1 % heads
        s = slot.get((b, head), 0)
        if s < len(R.PLANT_COORDS):
            R.plant(qkv, heads, fmt, base + 70, head, base + 3, [base + i for i in range(ln) if i != 3], 200.0, s)
    return planted


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("L", [8, 16, 32, 64, 128, 256, 384, 512])
def test_attention_dense(gpu_lib, fmt, L):
    heads = 12
    g = torch.Generator().manual_seed(L)
    pref = sorted({min(x, L) for x in (1, 31, 32, 33, 127, 128, 129, 255, 256, L)})
    lens = pref + [0, -1]                         # 0: all padding; -1: interior holes (the ids != 0 mask form)
    if L < 128:
        while (len(lens) * L) % 128 == 0 or (len(lens) * L // 128) < 1 or len(lens) % 2 == 0:
            lens.append(int(torch.randint(1, L + 1, (1,), generator=g)))
    B = len(lens)
    n = B * L
    qkv = R.random_qkv(n, heads, fmt, g)
    keep = torch.zeros(n, dtype=torch.bool)
    for b, ln in enumerate(lens):
        if ln == -1:
            keep[b * L:(b + 1) * L] = torch.rand(L, generator=g) < 0.7
            keep[b * L] = True
        else:
            keep[b * L:b * L + ln] = True
    planted = _plant_dense(qkv, heads, fmt, L, [int(keep[b * L:(b + 1) * L].sum()) if ln != -1 else 0 for b, ln in enumerate(lens)], 0)
    kbias = torch.where(keep, 0.0, -10000.0 * R.LOG2E).float().cuda()
    got = _run_attention(gpu_lib, fmt, _t16(qkv.cuda(), fmt), n, L, heads, kbias)
    lo = torch.arange(n) // L * L
    qkv_d, keep_d = qkv.cuda(), keep.cuda()
    ref, tol = R.attention_ref(qkv_d, heads, lo, lo + L, keep_d, fmt)
    k_ext, k_cut = keep.clone().view(B, L), keep.clone().view(B, L)
    for b, ln in enumerate(lens):
        if 0 < ln < L:
            k_ext[b, ln] = True
        if ln >= 2:
            k_cut[b, ln - 1] = False
    pert = {"key range +1": R.attention_ref(qkv_d, heads, lo, lo + L, k_ext.flatten().cuda(), fmt)[0],
            "last key masked": R.attention_ref(qkv_d, heads, lo, lo + L, k_cut.flatten().cuda(), fmt)[0]}
    if L > 128:
        pert["no alpha rescale"] = R.attention_no_rescale_ref(qkv_d, heads, L, keep_d)
        assert any(d > 8.0 for d in planted) and any(d < 8.0 for d in planted)
    _check(f"attention dense {fmt} L {L} B {B} planted {len(planted)}", got, ref, tol, pert)


def _pack(gpu_lib, lens, L, align):
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    B = len(lens)
    mt = 75776
    row0 = np.zeros(B, np.int32)
    lo = np.zeros(mt, np.int32)
    hi = np.zeros(mt, np.int32)
    tkv = np.zeros(2 * (mt // 128), np.int32)
    placed, tiles = C.c_int(), C.c_int()
    assert gpu_lib.ance_dbg_pack_packed(lens.ctypes.data, B, L, mt, align, row0.ctypes.data, lo.ctypes.data, hi.ctypes.data,
                                   tkv.ctypes.data, C.byref(placed), C.byref(tiles)) == 0, gpu_lib.ance_last_error()
    assert placed.value == B
    t = tiles.value
    return row0, lo[:t * 128], hi[:t * 128], tkv[:2 * t], t * 128


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("L", [64, 128, 256, 512])
@pytest.mark.parametrize("align", [1, 16])
def test_attention_packed(gpu_lib, fmt, L, align):
    """Row plans of ance_dbg_pack_packed (EDGE lengths of test_packed_plan.py mixed with random ones): every row against
    the fp64 attention over its own sequence only; peaked rows in long sequences that share warps with others."""
    heads = 12
    rng = np.random.default_rng(L + align)
    edge = [1, 16, 127, 128, 129, 255, 256, 384, 511, 512]
    lens = np.concatenate([np.minimum(edge, L), rng.integers(1, L + 1, 40)])
    lens = lens[rng.permutation(len(lens))]
    row0, lo, hi, tkv, n = _pack(gpu_lib, lens, L, align)
    g = torch.Generator().manual_seed(L * 3 + align)
    qkv = R.random_qkv(n, heads, fmt, g)
    planted = []
    for i in np.nonzero(lens > 128)[0][:6]:
        r0, ln = int(row0[i]), int(lens[i])
        for s, (r, d) in enumerate(((ln - 1, 30.0), (ln // 2, 8.1), (3, 120.0))):
            key = r0 + min(ln - 1, 128 + 40 * s)
            planted.append(R.plant(qkv, heads, fmt, r0 + r, s % heads, key, list(range(r0, r0 + 128)), d, s))
    kbias = torch.zeros(n, dtype=torch.float32, device="cuda")
    lo_t, hi_t = torch.from_numpy(lo).cuda(), torch.from_numpy(hi).cuda()
    tk = torch.from_numpy(tkv).cuda() if L > 128 else None
    got = _run_attention(gpu_lib, fmt, _t16(qkv.cuda(), fmt), n, L, heads, kbias, lo_t, hi_t, tk)
    qkv_d = qkv.cuda()
    lo64, hi64 = torch.from_numpy(lo).long(), torch.from_numpy(hi).long()
    ref, tol = R.attention_ref(qkv_d, heads, lo64, hi64, None, fmt)
    real = torch.zeros(n, dtype=torch.bool)
    for i in range(len(lens)):
        real[int(row0[i]):int(row0[i]) + int(lens[i])] = True
    ext = torch.where(real & (hi64 < n), hi64 + 1, hi64)
    cut = torch.where(real & (hi64 - lo64 >= 2), hi64 - 1, hi64)
    pert = {"key range +1": R.attention_ref(qkv_d, heads, lo64, ext, None, fmt)[0],
            "last key masked": R.attention_ref(qkv_d, heads, lo64, cut, None, fmt)[0]}
    _check(f"attention packed {fmt} L {L} align {align} tokens {n} planted {len(planted)}", got, ref, tol, pert,
           changed_rows=real.cuda())


# ------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------
def _run_ln(gpu_lib, fmt, x, in_f32, in_ld, rows, H, gam, bet, eps, out, rpw):
    kind = fmt if out == "16" else "f32"
    buf, view = _guarded(rows, H, kind)
    rc = gpu_lib.ance_dbg_layer_norm(FMT_CODE[fmt], x.data_ptr(), 1 if in_f32 else 0, in_ld, rows, H, gam.data_ptr(),
                                bet.data_ptr(), eps, view.data_ptr() if out == "16" else None,
                                view.data_ptr() if out == "32" else None, rpw, _st())
    assert rc == 0, gpu_lib.ance_last_error()
    torch.cuda.synchronize()
    _guards_intact(buf, rows, H)
    return view.to(F64)


def _ln_case(gpu_lib, fmt, rows, H, rpw, mode, seed, pitch=0, offset_rows=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    in_f32 = mode.startswith("32")
    ld = H + pitch
    x = torch.randn(rows, ld, generator=g, device="cuda", dtype=F64) * 0.05
    x[::3] *= 40.0
    if offset_rows:
        x[1::4] = 1e3 + torch.randn(x[1::4].shape, generator=g, device="cuda", dtype=F64) * 1e-2
    x = x.float() if in_f32 else _t16(x, fmt)
    xv = x[:, :H].to(F64)
    gam = (1.0 + 0.05 * torch.randn(H, generator=g, device="cuda")).float()
    bet = (0.05 * torch.randn(H, generator=g, device="cuda")).float()
    eps = 1e-5
    out = mode[-2:]
    got = _run_ln(gpu_lib, fmt, x, in_f32, ld, rows, H, gam, bet, eps, out, rpw)
    y, z = R.layer_norm_ref(xv, gam, bet, eps)
    tol = R.layer_norm_tol(xv, z, y, gam, bet, fmt if out == "16" else None)
    pert = {"unbiased var": R.layer_norm_ref(xv, gam, bet, eps, unbiased=True)[0],
            "eps outside sqrt": R.layer_norm_ref(xv, gam, bet, eps, eps_outside=True)[0]}
    small = torch.zeros(rows, dtype=torch.bool, device="cuda")
    small[1::3] = True                         # rows of std 0.05, where eps and the divisor show
    if offset_rows:
        small[1::4] = False
    if out == "16":   # 1/2 ulp16 (2^-11 / 2^-8 relative) hides the H - 1 divisor (1/(2H)), and in bf16 also eps
        pert = {} if fmt == "bf16" else {"eps outside sqrt": pert["eps outside sqrt"]}
    _check(f"layer norm {fmt} {mode} rows {rows} H {H} rpw {rpw} pitch {pitch} offset {offset_rows}", got, y, tol, pert,
           changed_rows=small, min_rows=1 if rows > 1 else 0)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("H", [256, 512, 768, 1024])
def test_layer_norm(gpu_lib, fmt, H):
    for rows in (1, 7, 4095, 4096, 4097, 38400):
        for rpw in ((1, 2, 3, 4) if H == 768 and rows >= 4096 else (2,)):
            _ln_case(gpu_lib, fmt, rows, H, rpw, "16to16", seed=rows + rpw + H)
        if rows in (1, 7, 4097):
            _ln_case(gpu_lib, fmt, rows, H, 2, "32to32", seed=rows * 3 + H)                    # the head LayerNorm
            _ln_case(gpu_lib, fmt, rows, H, 2, "32to32", seed=rows * 5 + H, offset_rows=True)  # 1e3 + N(0, 1e-2)
            _ln_case(gpu_lib, fmt, rows, H, 2, "16to32", seed=rows * 7 + H)
    _ln_case(gpu_lib, fmt, 4100, H, 2, "16to16", seed=H, pitch=3 * H)                            # rows at pitch 4H


@pytest.mark.parametrize("fmt", FMTS)
def test_layer_norm_constant_rows(gpu_lib, fmt):
    """Constant rows (exactly summable): the output is beta to one 16-bit ulp."""
    H, rows = 768, 4096
    c = torch.tensor([0.5, -3.25, 1e3, 0.0], dtype=F64, device="cuda").repeat(rows // 4)
    x = _t16(c[:, None].expand(rows, H).contiguous(), fmt)
    g = torch.Generator(device="cuda").manual_seed(0)
    gam = (1.0 + 0.05 * torch.randn(H, generator=g, device="cuda")).float()
    bet = (0.5 * torch.randn(H, generator=g, device="cuda")).float()
    for rpw in (1, 2, 3, 4):
        got = _run_ln(gpu_lib, fmt, x, False, H, rows, H, gam, bet, 1e-5, "16", rpw)
        d = (got - bet.double()).abs() / R.ulp16(bet.double(), fmt)
        assert d.max().item() <= 1.0, (rpw, d.max().item())


# ------------------------------------------------------------------------------------------------
# embeddings through ance_encoder_debug_hidden(0)
# ------------------------------------------------------------------------------------------------
def _backbone_encoder(sd, prefix, H, n_layer, ffn, vocab, max_pos, type_vocab, pad_id, eps, arch, fmt, max_tokens=8192):
    from ance_b200 import models
    bb = models._backbone(vocab, H, n_layer, ffn, max_pos, type_vocab, pad_id, eps)
    bb.load_state_dict({k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}, strict=True)
    return models._CudaEncoder(bb, arch, H // 64, pad_id, None, max_tokens, torch.device("cuda", torch.cuda.current_device()), fmt)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("H", [256, 512, 768, 1024])
@pytest.mark.parametrize("arch", ["roberta", "bert"])
def test_embeddings(gpu_lib, fmt, H, arch):
    from oracle.encoder_oracle import random_roberta_state_dict
    roberta = arch == "roberta"
    vocab, L = 1000, (512 if roberta else 256)
    max_pos, pad = (514, 1) if roberta else (512, 0)
    sd = random_roberta_state_dict(seed=H, n_layer=1, hidden=H, ffn=4 * H, vocab=vocab, max_pos=max_pos, head=False)
    enc = _backbone_encoder(sd, "roberta.", H, 1, 4 * H, vocab, max_pos, 1, pad, 1e-5,
                            _lib.ANCE_ARCH_ROBERTA if roberta else _lib.ANCE_ARCH_BERT, fmt)
    enc.enable_debug()
    g = torch.Generator().manual_seed(H)
    lens = torch.tensor([L, L - 1, 1, 200, 129, 37, 512, 2]).clamp(max=L)
    B = len(lens)
    ids = torch.randint(3, vocab, (B, L), generator=g, dtype=torch.int32)
    for b in range(B):
        ids[b, lens[b]:] = pad
    ids[0, 5], ids[1, 0] = vocab - 1, vocab - 1
    enc.forward(ids.cuda(), lens.to(torch.int32).cuda(), None)
    enc.check()
    got = enc.hidden(0, B * L).to(F64)
    w = {k[len("roberta."):]: v for k, v in sd.items()}
    x32, y, z = R.embed_ref(ids, w["embeddings.word_embeddings.weight"], w["embeddings.position_embeddings.weight"],
                          w["embeddings.token_type_embeddings.weight"], w["embeddings.LayerNorm.weight"],
                          w["embeddings.LayerNorm.bias"], 1e-5, roberta, pad)
    y, z = y.reshape(B * L, H).cuda(), z.reshape(B * L, H).cuda()
    gam, bet = w["embeddings.LayerNorm.weight"].cuda(), w["embeddings.LayerNorm.bias"].cuda()
    tol = R.layer_norm_tol(x32.reshape(B * L, H).cuda(), z, y, gam, bet, fmt)
    if roberta:
        assert int(R.position_ids(ids.long(), True, pad).max()) == max_pos - 1
    pos_shift = R.position_ids(ids.long(), roberta, pad) + 1
    xs = (w["embeddings.word_embeddings.weight"][ids.long()] + w["embeddings.position_embeddings.weight"][
        pos_shift.clamp(max=max_pos - 1)]) + w["embeddings.token_type_embeddings.weight"][0]
    pert = {"position + 1": R.layer_norm_ref(xs.reshape(B * L, H).cuda(), gam, bet, 1e-5)[0]}
    _check(f"embeddings {arch} {fmt} H {H} L {L}", got, y, tol, pert, min_rows=B * L // 2)


# ------------------------------------------------------------------------------------------------
# end to end against the fp32 oracle (the 0.03 gate of test_gpu_encoder.py), layer by layer
# ------------------------------------------------------------------------------------------------
MAXABS = 0.03


def _oracle_layers(sd, prefix, arch, n_layer, heads, pad, eps, ids, mask):
    from oracle.encoder_oracle import EncoderOracle
    return EncoderOracle(sd, prefix, arch, n_layer, heads, pad, eps, device="cuda").hidden_states(ids, mask)


@pytest.mark.parametrize("H", [256, 1024])
def test_small_and_large_hidden_layer_by_layer(gpu_lib, H):
    """2-layer encoders at hidden 256 (4 heads) and 1024 (16 heads), every hidden state against the fp32 oracle."""
    from oracle.encoder_oracle import random_roberta_state_dict
    vocab = 5000
    sd = random_roberta_state_dict(seed=H, n_layer=2, hidden=H, ffn=4 * H, vocab=vocab, max_pos=514, head=False)
    enc = _backbone_encoder(sd, "roberta.", H, 2, 4 * H, vocab, 514, 1, 1, 1e-5, _lib.ANCE_ARCH_ROBERTA, "fp16")
    enc.enable_debug()
    enc.set_param("prune_last_layer", 0)
    g = torch.Generator().manual_seed(1)
    B, L = 12, 128
    ids = torch.randint(3, vocab, (B, L), generator=g, dtype=torch.int32)
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[0] = L
    for b in range(B):
        ids[b, lens[b]:] = 1
    mask = torch.arange(L)[None, :] < lens[:, None]
    out = enc.forward(ids.cuda(), lens.to(torch.int32).cuda(), None)
    enc.check()
    hs = _oracle_layers(sd, "roberta.", "roberta", 2, H // 64, 1, 1e-5, ids, mask)
    m = mask.reshape(-1).cuda()
    for l in range(3):
        d = (enc.hidden(l, B * L) - hs[l].reshape(B * L, H)).abs()[m].max().item()
        print(f"hidden {H} layer {l}: max |diff| {d:.4f}")
        assert d <= MAXABS, (H, l, d)
    assert (out - hs[2][:, 0]).abs().max().item() <= MAXABS


def test_peaked_attention_end_to_end(gpu_lib):
    """A 2-layer RoBERTa with query weights scaled so that attention is peaked (score std >= 6 nats), at L = 512:
    dense layer by layer, and dense / packed exact / packed densest embeddings, against the fp32 oracle."""
    from ance_b200.models import RobertaDot_NLL_LN
    from oracle.encoder_oracle import RobertaDotOracle, random_roberta_state_dict
    from transformers import RobertaConfig
    sd = random_roberta_state_dict(seed=3, n_layer=2)
    for l in range(2):
        sd[f"roberta.encoder.layer.{l}.attention.self.query.weight"] *= 8.0
    cfg = RobertaConfig(vocab_size=50265, hidden_size=768, num_hidden_layers=2, num_attention_heads=12,
                        intermediate_size=3072, max_position_embeddings=514, type_vocab_size=1, layer_norm_eps=1e-5,
                        pad_token_id=1, bos_token_id=0, eos_token_id=2)
    m = RobertaDot_NLL_LN(cfg)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    g = torch.Generator().manual_seed(2)
    B, L = 8, 512
    lens = torch.tensor([512, 129, 300, 1, 511, 256, 77, 400])
    ids = torch.randint(3, 50265, (B, L), generator=g, dtype=torch.int32)
    for b in range(B):
        ids[b, lens[b]:] = 1
    ids[:, 0] = 0
    mask = torch.arange(L)[None, :] < lens[:, None]
    orc = RobertaDotOracle(sd, n_layer=2, device="cuda")
    hs = orc.enc.hidden_states(ids, mask)
    # the scores of layer 0 really are peaked
    x0 = hs[0][0, :lens[0]].double()
    wq = sd["roberta.encoder.layer.0.attention.self.query.weight"].double().cuda()
    wk = sd["roberta.encoder.layer.0.attention.self.key.weight"].double().cuda()
    q = (x0 @ wq.T).view(-1, 12, 64).transpose(0, 1)
    k = (x0 @ wk.T).view(-1, 12, 64).transpose(0, 1)
    std = (q @ k.transpose(1, 2) / 8.0).std().item()
    print(f"peaked layer-0 score std {std:.2f} nats")
    assert std >= 6.0
    enc = m._encoder(torch.device("cuda", torch.cuda.current_device()))
    enc.enable_debug()
    ids_d, lens_d = ids.cuda(), lens.to(torch.int32).cuda()
    dense = m.encode_lens(ids_d, lens_d)
    mk = mask.reshape(-1).cuda()
    for l in range(2):
        d = (enc.hidden(l, B * L) - hs[l].reshape(B * L, -1)).abs()[mk].max().item()
        print(f"peaked layer {l}: max |diff| {d:.4f}")
        assert d <= MAXABS, (l, d)
    ref = orc.query_emb(ids, mask)
    exact = enc.forward_packed(ids_d, lens_d, lens_host=lens.to(torch.int32), align=16)
    densest = enc.forward_packed(ids_d, lens_d, lens_host=lens.to(torch.int32), align=1)
    for name, e in (("dense", dense), ("packed exact", exact), ("packed densest", densest)):
        d = (e - ref).abs().max().item()
        print(f"peaked {name}: max |diff| {d:.4f}")
        assert d <= MAXABS, (name, d)
    assert torch.equal(exact, dense)
