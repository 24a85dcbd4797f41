"""The 128 x 256 two-warpgroup GEMM (ance_dbg_gemm variant 5, tc05_gemm_wide_kernel) against the 128 x 128 tile
(variant 0): with a 16-bit output the two compute the same per-element arithmetic in the same order, so the outputs
must be torch.equal, in fp16 and bf16 operands, with and without bias and residual (and both GELU forms at N 3072).
Shapes cover the four encoder layer shapes, M not a multiple of 128 (and a last tile whose second 64-row half is
empty), fewer tiles than SMs, N a multiple of 8 but not of 256, K not a multiple of 64, and several tiles per CTA.
Output buffers carry guard rows that must survive.  The last test runs linear() (ance_dbg_linear) at sizes that take
the wide kernel, with the strided A and residual rows of the encoder's calls, against variant 0 on contiguous
copies."""
import pytest
import torch

from ance_b200 import _lib

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
