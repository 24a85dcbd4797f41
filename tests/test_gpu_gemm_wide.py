"""The 128 x 256 two-warpgroup GEMM (ance_dbg_gemm variant 5, tc05_gemm_wide_kernel) against the 128 x 128 tile
(variant 0): with a 16-bit output the two compute the same per-element arithmetic in the same order, so the outputs
must be torch.equal, in fp16 and bf16 operands, with and without bias and residual (and both GELU forms at N 3072).
Shapes cover the four encoder layer shapes, M not a multiple of 128 (and a last tile whose second 64-row half is
empty), fewer tiles than SMs, N a multiple of 8 but not of 256, K not a multiple of 64, and several tiles per CTA.
Output buffers carry guard rows that must survive.  The ance_dbg_gemm hook runs EpStoreWide<> (bf16 output and
residual) whatever the operand format.

The remaining tests run linear() (ance_dbg_linear), i.e. the encoder's own instantiations EpStoreWide<kFmtF16> and
<kFmtBF16> (output and residual in the operand format), at the sizes where linear() routes to the wide kernel:
  - the routing itself, read from the kernel names under torch.profiler (in a child process), on both sides of the
    threshold;
  - every routed call against fp64 (encoder_refs.linear_discrimination_blocked) with perturbed references that a
    two-warpgroup 128 x 256 tile could produce, which must be rejected;
  - every routed call bit-identical to the same call cut into row slices that stay below the threshold (128 x 128
    tile), with the strided A and residual rows of the encoder's calls.
The threshold is computed from the device's SM count with linear()'s formula, and every case asserts which side of
it its calls are on, so a change of the threshold cannot quietly leave a routed case unrouted."""
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from ance_b200 import _lib
from tests import encoder_refs as ER

pytestmark = pytest.mark.gpu

FMTS = ["fp16", "bf16"]
FMT_CODE = {"fp16": _lib.ANCE_FMT_FP16, "bf16": _lib.ANCE_FMT_BF16}
DT = {"fp16": torch.float16, "bf16": torch.bfloat16}
GUARD = 64
SENT16 = 0x7E5A   # a NaN in bf16

SHAPES = [
    (1000, 2304, 768), (1000, 768, 768), (1000, 3072, 768), (1000, 768, 3072),   # layer shapes, small M
    (4161, 768, 768), (64, 768, 768), (1, 776, 768), (300, 768, 3072),           # ragged M, fewer tiles than SMs
    (700, 776, 768), (2000, 2312, 768), (513, 8, 64),                            # N % 256 != 0
    (900, 768, 200), (600, 2304, 40), (257, 776, 776),                           # K % 64 != 0
    (8192, 3072, 768), (20000, 768, 768),                                        # several tiles per CTA
]


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available()
    return _lib.load()


def _guarded(rows, cols):
    buf = torch.full(((rows + 2 * GUARD) * cols,), SENT16, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    return buf, buf[GUARD * cols:(GUARD + rows) * cols].view(rows, cols)


def _gemm(lib, variant, fmt, A, W, bias, R, act=0):
    M, K = A.shape
    N = W.shape[0]
    buf, out = _guarded(M, N)
    rc = lib.ance_dbg_gemm(A.data_ptr(), W.data_ptr(), M, N, K, FMT_CODE[fmt], variant,
                           None if bias is None else bias.data_ptr(), None if R is None else R.data_ptr(), act,
                           out.data_ptr(), None, _lib.current_stream())
    assert rc == 0, lib.ance_last_error()
    torch.cuda.synchronize()
    raw = buf.view(torch.int16)
    assert bool((raw[:GUARD * N] == SENT16).all()) and bool((raw[(GUARD + M) * N:] == SENT16).all()), \
        f"variant {variant}: a guard row was overwritten"
    return out


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("MNK", SHAPES, ids=lambda s: "M%d_N%d_K%d" % s)
def test_wide_equals_128x128(lib, fmt, MNK):
    """Variant 5 against variant 0.  Both run with a bf16 output and a bf16 residual in either operand format, so the
    "fp16" case is fp16 operands with a bf16 output (linear()'s fp16 instantiation is tested below)."""
    M, N, K = MNK
    g = torch.Generator(device="cuda").manual_seed(M * 31 + N * 7 + K)
    A = torch.randn(M, K, generator=g, device="cuda").to(DT[fmt])
    W = (torch.randn(N, K, generator=g, device="cuda") * 0.04).to(DT[fmt])
    bias = torch.randn(N, generator=g, device="cuda")
    R = torch.randn(M, N, generator=g, device="cuda").to(torch.bfloat16)
    for act in ((0, 1, 2) if N == 3072 else (0,)):
        for b in (None, bias):
            for r in (None, R):
                ref = _gemm(lib, 0, fmt, A, W, b, r, act)
                got = _gemm(lib, 5, fmt, A, W, b, r, act)
                assert not bool(torch.isnan(ref).any())
                assert torch.equal(got, ref), (fmt, MNK, act, b is not None, r is not None,
                                               (got.float() - ref.float()).abs().max().item())


def test_wide_refuses_fp32_output(lib):
    A = torch.zeros(256, 64, device="cuda", dtype=torch.float16)
    W = torch.zeros(256, 64, device="cuda", dtype=torch.float16)
    C32 = torch.empty(256, 256, device="cuda")
    st = _lib.current_stream()
    assert lib.ance_dbg_gemm(A.data_ptr(), W.data_ptr(), 256, 256, 64, FMT_CODE["fp16"], 5, None, None, 0,
                             None, C32.data_ptr(), st) != 0


@pytest.mark.parametrize("case", [(60000, 768, 768, 768, 768), (24000, 2304, 768, 768, 2304),
                                  (57000, 768, 3072, 3072, 768), (60000, 768, 768, 2 * 768, 3 * 768)],
                         ids=["out", "qkv", "ffn2", "strided"])
def test_linear_takes_wide_bit_identical(lib, case):
    """linear() with a bf16 output, act 0 and enough tiles to take the wide kernel (at least 10 per SM on a 132-SM
    H100), with and without residual, equals the 128 x 128 tile (variant 0, bf16 output and residual) on contiguous
    copies of the same operands."""
    M, N, K, lda, ldr = case
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    Abuf = torch.randn((M - 1) * lda + K, generator=g, device="cuda").to(torch.bfloat16)
    A = Abuf.as_strided((M, K), (lda, 1))
    W = (torch.randn(N, K, generator=g, device="cuda") * 0.04).to(torch.bfloat16)
    bias = torch.randn(N, generator=g, device="cuda")
    Rbuf = torch.randn((M - 1) * ldr + N, generator=g, device="cuda").to(torch.bfloat16)
    Rv = Rbuf.as_strided((M, N), (ldr, 1))
    for res in (False, True):
        buf, out = _guarded(M, N)
        rc = lib.ance_dbg_linear(FMT_CODE["bf16"], Abuf.data_ptr(), lda, M, W.data_ptr(), N, K, bias.data_ptr(),
                                 Rbuf.data_ptr() if res else None, ldr if res else 0, 0, out.data_ptr(), None,
                                 _lib.current_stream())
        assert rc == 0, lib.ance_last_error()
        torch.cuda.synchronize()
        raw = buf.view(torch.int16)
        assert bool((raw[:GUARD * N] == SENT16).all()) and bool((raw[(GUARD + M) * N:] == SENT16).all())
        ref = _gemm(lib, 0, "bf16", A.contiguous(), W, bias, Rv.contiguous() if res else None)
        assert torch.equal(out, ref), (case, res, (out.float() - ref.float()).abs().max().item())


# ------------------------------------------------------------------------------------------------
# linear() at the sizes that route to the wide kernel
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def threshold():
    return ER.wide_threshold(torch.cuda.get_device_properties(0).multi_processor_count)


def _routed_m(N, thr):
    """Fewest rows of an [M, N] call that take the wide kernel (its last 128-row tile holds one row)."""
    return (-(-thr // -(-N // 256)) - 1) * 128 + 1


def _linear16(lib, fmt, Abuf, lda, M, W, N, K, bias, Rbuf, ldr, act=0, out=None):
    """ance_dbg_linear with a 16-bit output (into `out` [M, N] when given, else a guarded buffer whose guards are
    checked) -> out."""
    buf = None
    if out is None:
        buf, out = _guarded(M, N)
        out = out.view(DT[fmt])
    rc = lib.ance_dbg_linear(FMT_CODE[fmt], Abuf.data_ptr(), lda, M, W.data_ptr(), N, K,
                             None if bias is None else bias.data_ptr(), None if Rbuf is None else Rbuf.data_ptr(),
                             ldr if Rbuf is not None else 0, act, out.data_ptr(), None, _lib.current_stream())
    assert rc == 0, lib.ance_last_error()
    if buf is not None:
        torch.cuda.synchronize()
        raw = buf.view(torch.int16)
        assert bool((raw[:GUARD * N] == SENT16).all()) and bool((raw[(GUARD + M) * N:] == SENT16).all()), \
            "a guard row was overwritten"
    return out


def _routing_kernels():
    """Child-process half of test_linear_routing_at_the_threshold: runs each call under torch.profiler and prints one
    JSON line [[fmt, M, N, act, output, kernel], ...], kernel "wide" (tc05_gemm_wide_kernel), "128x128"
    (tc05_gemm_kernel) or the name of whatever else ran."""
    import json
    from torch.profiler import ProfilerActivity, profile
    lib = _lib.load()
    thr = ER.wide_threshold(torch.cuda.get_device_properties(0).multi_processor_count)
    N = K = 768
    M_big = 75776
    # one set of 16-bit buffers for both formats: only the kernel that runs is read here, not the values
    g = torch.Generator(device="cuda").manual_seed(3)
    A = torch.randn(M_big, 3072, generator=g, device="cuda").to(torch.float16)
    W = (torch.randn(3072, 3072, generator=g, device="cuda") * 0.04).to(torch.float16)
    bias = torch.randn(3072, generator=g, device="cuda")
    C16 = torch.empty(M_big * 3072, device="cuda", dtype=torch.float16)
    C32 = torch.empty(M_big * 768, device="cuda")
    calls = []
    for fmt in FMTS:
        calls += [(fmt, M, N, K, 0, "c16") for M in (ER.wide_slice_rows(N, thr), _routed_m(N, thr))]
        calls += [(fmt, M_big, 3072, 768, act, "c16") for act in (1, 2)]   # the FFN-up shape with GELU
        calls += [(fmt, M, N, K, 0, "c32") for M in (_routed_m(N, thr), M_big)]
    rows = []
    for fmt, M, n, k, act, out in calls:
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            rc = lib.ance_dbg_linear(FMT_CODE[fmt], A.data_ptr(), k, M, W.data_ptr(), n, k, bias.data_ptr(), None, 0,
                                     act, C16.data_ptr() if out == "c16" else None,
                                     C32.data_ptr() if out == "c32" else None, _lib.current_stream())
            torch.cuda.synchronize()
        assert rc == 0, lib.ance_last_error()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        kern = ["wide" if "tc05_gemm_wide_kernel" in x else "128x128" if "tc05_gemm_kernel" in x else x for x in names]
        rows.append([fmt, M, n, act, out, kern[0] if len(kern) == 1 else kern])
    print(json.dumps(rows))


def test_linear_routing_at_the_threshold(threshold):
    """linear() runs tc05_gemm_wide_kernel from threshold tiles on and tc05_gemm_kernel below; GELU (act 1, 2) and an
    fp32 output never take the wide kernel, at any size.  The kernel names come from torch.profiler in a child process,
    so that this test leaves no profiler state behind: after sessions here and the host-index tests, a later session
    in the same process (test_gpu_lamb.py reads kernel names too) has been seen to record no GPU activity."""
    N = 768
    M_hi, M_lo = _routed_m(N, threshold), ER.wide_slice_rows(N, threshold)
    assert ER.wide_tiles(M_lo, N) < threshold <= ER.wide_tiles(M_hi, N) and M_hi % 128 == 1 and M_lo == M_hi - 1
    assert ER.wide_tiles(75776, 3072) >= 2 * threshold
    root = Path(__file__).resolve().parent.parent
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(root)] + [os.environ.get("PYTHONPATH", "")]))
    r = subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c",
                        "from tests.test_gpu_gemm_wide import _routing_kernels; _routing_kernels()"],
                       cwd=root, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    rows = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(rows) == 12
    for fmt, M, n, act, out, kern in rows:
        print(f"linear {fmt} M{M} N{n} act {act} {out}: {ER.wide_tiles(M, n)} tiles, threshold {threshold} -> {kern}")
        routed = out == "c16" and act == 0 and ER.wide_tiles(M, n) >= threshold
        assert kern == ("wide" if routed else "128x128"), (fmt, M, n, act, out, kern)
    assert sum(kern == "wide" for *_, kern in rows) == 2 and {M for _, M, *_ in rows} >= {M_lo, M_hi}


# (name, M, N, K, bias, residual, lda, ldr): the four layer calls of one flagship encoder pass (75,776 rows), then the
# edges at routed M (None = the fewest routed rows at that N on this device).
ROUTED = [
    ("qkv", 75776, 2304, 768, True, False, 768, 0),
    ("out_proj", 75776, 768, 768, True, True, 768, 768),
    ("ffn_up_copy", 75776, 3072, 768, True, False, 768, 0),
    ("ffn_down", 75776, 768, 3072, True, True, 3072, 768),
    ("boundary", None, 768, 768, True, True, 768, 768),               # last tile: 1 row
    ("last_tile_64", 440 * 128 + 64, 768, 768, True, True, 768, 768),  # second warpgroup's half empty
    ("last_tile_65", 440 * 128 + 65, 768, 768, True, True, 768, 768),  # ... holding one row
    ("n776", None, 776, 768, True, True, 768, 776),                  # partial 256-column block and 64-column slab
    ("strided", 60000, 768, 768, True, True, 3 * 768, 3 * 768),        # the encoder's strided A and residual rows
]
ROUTED_IDS = [c[0] for c in ROUTED]


def _routed_case(lib, fmt, case, threshold):
    """Operands of a routed case in the operand format, the routed output, and the call's shape."""
    name, M, N, K, bias_on, res_on, lda, ldr = case
    M = M or _routed_m(N, threshold)
    tiles = ER.wide_tiles(M, N)
    print(f"{name} {fmt}: M{M} N{N} K{K}: {tiles} wide tiles, threshold {threshold}")
    assert tiles >= threshold, (name, tiles, threshold)
    g = torch.Generator(device="cuda").manual_seed(M + 3 * N + 7 * K + (fmt == "bf16"))
    Abuf = torch.randn((M - 1) * lda + K, generator=g, device="cuda").to(DT[fmt])
    W = (torch.randn(N, K, generator=g, device="cuda") * 0.04).to(DT[fmt])
    bias = torch.randn(N, generator=g, device="cuda") if bias_on else None
    Rbuf = torch.randn((M - 1) * ldr + N, generator=g, device="cuda").to(DT[fmt]) if res_on else None
    out = _linear16(lib, fmt, Abuf, lda, M, W, N, K, bias, Rbuf, ldr)
    return M, N, K, lda, ldr, Abuf, W, bias, Rbuf, out


def _check_fp64(name, out, A, W, bias, Rv, fmt):
    err, rep = ER.linear_discrimination_blocked(out, A, W, bias, Rv, fmt)
    print(f"{name}: max err / bound {err:.3f}; perturbed (fraction rejected, median margin, rows) {rep}")
    assert err <= 1.0, (name, err)
    M = out.shape[0]
    for k, (frac, margin, rows) in rep.items():
        assert rows >= M // 2 and frac == 1.0, (name, k, rep[k])


def _check_slices(lib, fmt, name, out, M, N, K, lda, ldr, Abuf, W, bias, Rbuf, threshold):
    """The routed output equals the call cut into row slices below the threshold (A, residual and C offset by each
    slice's first row)."""
    step = ER.wide_slice_rows(N, threshold)
    assert ER.wide_tiles(step, N) < threshold
    cut = torch.empty_like(out)
    for r0 in range(0, M, step):
        m = min(step, M - r0)
        _linear16(lib, fmt, Abuf[r0 * lda:], lda, m, W, N, K, bias, None if Rbuf is None else Rbuf[r0 * ldr:], ldr,
                  out=cut[r0:r0 + m])
    torch.cuda.synchronize()
    same = torch.equal(out, cut)
    print(f"{name}: bit-identical to {-(-M // step)} slices of <= {step} rows (128 x 128 tile): {same}")
    assert same, (name, (out.float() - cut.float()).abs().max().item())


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("case", ROUTED, ids=ROUTED_IDS)
def test_linear_routed_fp64_and_slices(lib, fmt, case, threshold):
    """One routed call of EpStoreWide<FMT>: within the fp64 bound, every perturbed reference rejected, and bit-identical
    to the 128 x 128 tile on row slices below the threshold."""
    M, N, K, lda, ldr, Abuf, W, bias, Rbuf, out = _routed_case(lib, fmt, case, threshold)
    A = Abuf.as_strided((M, K), (lda, 1))
    Rv = None if Rbuf is None else Rbuf.as_strided((M, N), (ldr, 1))
    name = f"{case[0]} {fmt} M{M} N{N} K{K} lda{lda} ldr{ldr}"
    _check_fp64(name, out, A, W, bias, Rv, fmt)
    _check_slices(lib, fmt, name, out, M, N, K, lda, ldr, Abuf, W, bias, Rbuf, threshold)


def test_linear_routed_dgrad_shape(lib, threshold):
    """The backward's dgrad into CTX (bf16, no bias, no residual, 16-bit output) at 448 x 128 tokens."""
    case = ("dgrad", 57344, 768, 768, False, False, 768, 0)
    M, N, K, lda, ldr, Abuf, W, bias, Rbuf, out = _routed_case(lib, "bf16", case, threshold)
    name = f"dgrad bf16 M{M} N{N} K{K}"
    _check_fp64(name, out, Abuf.view(M, K), W, None, None, "bf16")
    _check_slices(lib, "bf16", name, out, M, N, K, lda, ldr, Abuf, W, None, None, threshold)
