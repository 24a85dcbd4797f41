"""fp64 references of the encoder kernels, their error models, and perturbed references (test infrastructure only).

Every reference takes the SAME 16-bit operands the kernel reads (as float tensors holding 16-bit values), so operand
rounding is not counted as kernel error.  Each family comes with a per-element tolerance derived from a written error
model (the docstrings below), not fitted to measurements, and with perturbed references: the outputs plausible kernel
bugs would produce.  The tests require the kernels inside the tolerance of the reference and outside it of every
perturbed one.  Everything here is plain torch fp64 and runs on the CPU or on a CUDA device alike.
"""
from __future__ import annotations

import math
import re
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
LOG2E = 1.4426950408889634
F64 = torch.float64

# |GELU form - erf-GELU| in fp32 with exactly rounded exp / reciprocal (measured over |x| <= 1e4 by
# test_encoder_refs_cpu.py::test_gelu_forms_within_documented_bounds; documented in gemm_store.cuh and DESIGN.md 4.1)
GELU_BOUND = {1: 7.1e-7, 2: 3.7e-6}
# ex2.approx.ftz / rcp.approx.ftz relative error allowance (PTX ISA: ex2.approx.f32 <= 2^-22.5 relative near 1 and
# rcp.approx.f32 <= 1 ulp; both rounded up to 2^-21 here)
APPROX_REL = 2.0 ** -21
U32 = 2.0 ** -24   # unit roundoff of fp32


def dtype16(fmt: str):
    return {"fp16": torch.float16, "bf16": torch.bfloat16}[fmt]


def round16(x: torch.Tensor, fmt: str) -> torch.Tensor:
    """Round to the 16-bit format and back to fp64 (round to nearest even)."""
    return x.to(dtype16(fmt)).to(F64)


def ulp16(x: torch.Tensor, fmt: str) -> torch.Tensor:
    """Spacing of the 16-bit format at |x| (subnormal spacing below the smallest normal)."""
    man, emin = (10, -14) if fmt == "fp16" else (7, -126)
    a = x.abs().to(F64).clamp_min(2.0 ** emin)
    return torch.exp2(torch.floor(torch.log2(a)).clamp_min(emin) - man)


def half_u16(fmt: str) -> float:
    """Relative rounding error bound of the 16-bit format (normal range)."""
    return 2.0 ** -11 if fmt == "fp16" else 2.0 ** -8


def gelu_erf(x: torch.Tensor) -> torch.Tensor:
    """Exact GELU x * Phi(x) in fp64 (torch.special.erf in fp64; tied to scipy.special.erf by the CPU tests)."""
    x = x.to(F64)
    return 0.5 * x * (1.0 + torch.special.erf(x / math.sqrt(2.0)))


def gelu_tanh(x: torch.Tensor) -> torch.Tensor:
    """The tanh approximation (HF "gelu_new"): a plausible wrong GELU."""
    x = x.to(F64)
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


# ------------------------------------------------------------------------------------------------
# GEMM epilogue
# ------------------------------------------------------------------------------------------------
def linear_ref(A, W, bias=None, R=None, act=0, gelu=gelu_erf, bias_shift=0, res_shift=0):
    """C = act(A W^T + bias) + R in fp64.  act 1 / 2 (either GELU form of the kernel) -> exact erf-GELU.
    Perturbations: `gelu` (e.g. gelu_tanh), `bias_shift` = 1 (bias of column n + 1), `res_shift` = 1 (residual of the
    next row, i.e. an off-by-one residual pitch)."""
    x = A.to(F64) @ W.to(F64).T
    if bias is not None:
        b = bias.to(F64)
        if bias_shift:
            b = torch.cat([b[bias_shift:], b[:bias_shift]])
        x = x + b
    y = gelu(x) if act else x
    if R is not None:
        r = R.to(F64)
        if res_shift:
            r = torch.cat([r[res_shift:], r[:res_shift]])
        y = y + r
    return x, y


def linear_tol(A, W, x, y, R, act, out_fmt):
    """Error model of one output element of linear<FMT> (out_fmt None = fp32 output C32):
      accumulation  K * 2^-22 * sum_k |a_k w_k|        (the search certificate's term: at most one ulp of the largest
                                                        partial sum per addition, with 2x margin; Sigma|a w| instead of
                                                        |a||w|, which bounds every partial sum just as well)
      bias add      2^-24 |x|
      GELU          (above) * 1.13 (max |GELU'|) + GELU_BOUND[act] + 4 * APPROX_REL * |x|   (ex2 / rcp approximations)
      residual add  2^-24 (|y| + |r|)
      output        1/2 ulp16(|y| + delta) for a 16-bit output"""
    K = A.shape[1]
    acc = K * 2.0 ** -22 * (A.to(F64).abs() @ W.to(F64).abs().T) + U32 * x.abs()
    if act:
        d = 1.13 * acc + GELU_BOUND[act] + 4 * APPROX_REL * x.abs()
    else:
        d = acc
    if R is not None:
        d = d + U32 * (y.abs() + R.to(F64).abs())
    d = d + U32 * y.abs()
    if out_fmt is not None:
        d = d + 0.5 * ulp16(y.abs() + d, out_fmt)
    return d


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def _ranges(lo, hi):
    lo = torch.as_tensor(lo, dtype=torch.int64)
    hi = torch.as_tensor(hi, dtype=torch.int64)
    pairs = torch.stack([lo, hi], 1)
    uniq, inv = torch.unique(pairs, dim=0, return_inverse=True)
    return uniq.tolist(), inv


def attention_ref(qkv, heads, lo, hi, keep=None, fmt="fp16"):
    """ctx = softmax(Q K^T / 8 + mask) V per row over the keys [lo[r], hi[r]) of its own sequence, in fp64.

    keep [n_tokens] bool (None: every key kept): a masked key's score follows HF-2.3.0's fp32 arithmetic,
    fl32(fl32(s) - 10000), so that an all-padding row keeps the reference's finite "uniform" value.
    Returns (out [n, 64 heads], tol [n, 64 heads]) with the error model of attention_kernel:
      per key, relative error of p_j:  score  2^-17 sum_i |q_i k_i| / 8 (fp32 accumulation of 64 exact products)
                                              + 2^-22 (|t_j| + |m|) ln 2 (fp32 rounding of t = s log2e / 8 and t - m)
                                              + 2^-10 for an all-padding row (ulp32(10000) of the masked scores)
                                       ex2    APPROX_REL
      tol = (1/2 u16 [P rounded to 16 bits; the row sums are not] + 2 (score + ex2) [numerator and denominator]
             + n 2^-22 [P V accumulation] + n 2^-23 [row sum]) * sum_j p_j |v_j| / l
            + n 2^-25 max |v| (fp16 only: P below 2^-14 is subnormal)  + 1/2 ulp16(|out| + delta)."""
    qkv = qkv.to(F64)
    n = qkv.shape[0]
    H = heads * 64
    out = torch.zeros(n, H, dtype=F64, device=qkv.device)
    tol = torch.zeros(n, H, dtype=F64, device=qkv.device)
    if keep is None:
        keep = torch.ones(n, dtype=torch.bool, device=qkv.device)
    keep = torch.as_tensor(keep, device=qkv.device).bool()
    uniq, inv = _ranges(lo, hi)
    inv = inv.to(qkv.device)
    for g, (a, b) in enumerate(uniq):
        rows = torch.nonzero(inv == g).flatten()
        q = qkv[rows, :H].view(-1, heads, 64).transpose(0, 1)            # [h, r, 64]
        k = qkv[a:b, H:2 * H].view(-1, heads, 64).transpose(0, 1)        # [h, n, 64]
        v = qkv[a:b, 2 * H:].view(-1, heads, 64).transpose(0, 1)
        s = q @ k.transpose(1, 2) / 8.0
        sabs = q.abs() @ k.abs().transpose(1, 2) / 8.0
        kp = keep[a:b]
        all_pad = not bool(kp.any())
        if not bool(kp.all()):
            sm = (s.float() - 10000.0).to(F64)
            s = torch.where(kp[None, None, :], s, sm)
        p = torch.softmax(s, dim=-1)
        o = p @ v
        W = p @ v.abs()
        # error model
        t = s * LOG2E
        m = t.max(dim=-1, keepdim=True).values
        real = kp[None, None, :] if not all_pad else torch.ones_like(kp)[None, None, :]
        es = torch.where(real, 2.0 ** -17 * sabs + 2.0 ** -22 * (t.abs() + m.abs()) * math.log(2.0), torch.zeros_like(s))
        es = es.max(dim=-1, keepdim=True).values + (2.0 ** -10 if all_pad else 0.0)
        nk = b - a
        rel = half_u16(fmt) + 2 * (es + APPROX_REL) + nk * 2.0 ** -22 + nk * 2.0 ** -23
        d = rel * W
        if fmt == "fp16":
            d = d + nk * 2.0 ** -25 * v.abs().amax(dim=(1, 2))[:, None, None]
        d = d + 0.5 * ulp16(o.abs() + d, fmt)
        out[rows] = o.transpose(0, 1).reshape(-1, H)
        tol[rows] = d.transpose(0, 1).reshape(-1, H)
    return out, tol


def attention_no_rescale_ref(qkv, heads, L, keep):
    """Perturbed reference: dense sequences of L > 128 tokens, the online softmax over 128-key blocks with the kernel's
    optimistic rule (a later block is rescaled only when it raises the row maximum by more than 8 log2 units), but the
    running output NOT multiplied by alpha when it is (the row sum is).  fp64."""
    qkv = qkv.to(F64)
    n = qkv.shape[0]
    H = heads * 64
    out = torch.zeros(n, H, dtype=F64, device=qkv.device)
    keep = torch.as_tensor(keep, device=qkv.device).bool()
    for a in range(0, n, L):
        q = qkv[a:a + L, :H].view(-1, heads, 64).transpose(0, 1)
        k = qkv[a:a + L, H:2 * H].view(-1, heads, 64).transpose(0, 1)
        v = qkv[a:a + L, 2 * H:].view(-1, heads, 64).transpose(0, 1)
        s = q @ k.transpose(1, 2) / 8.0
        kp = keep[a:a + L]
        s = torch.where(kp[None, None, :], s, (s.float() - 10000.0).to(F64))
        t = s * LOG2E
        m_run = t[..., :128].max(-1, keepdim=True).values
        pb = torch.exp2(t[..., :128] - m_run)
        o = pb @ v[:, :128]
        l = pb.sum(-1, keepdim=True)
        for j in range(128, L, 128):
            tb = t[..., j:j + 128]
            over = (tb - m_run).max(-1, keepdim=True).values
            redo = over > 8.0
            m_new = torch.where(redo, m_run + over, m_run)
            alpha = torch.exp2(m_run - m_new)
            pb = torch.exp2(tb - m_new)
            o = o + pb @ v[:, j:j + 128]            # the bug: o * alpha missing
            l = l * alpha + pb.sum(-1, keepdim=True)
            m_run = m_new
        out[a:a + L] = (o / l).transpose(0, 1).reshape(-1, H)
    return out


def attention_emulate(qkv16, heads, L, keep, fmt):
    """fp32 emulation of attention_kernel's arithmetic on dense sequences of L tokens (L a multiple of 128, or a divisor
    of 128 with one block): fp32 scores t = fl32(s log2e/8 + bias), per 128-key block the kernel's online softmax
    (first block: two passes, later blocks: one pass relative to the running maximum, redone relative to the true one when
    any row of the 32-row warp sees a score more than 8 log2 units above it), P rounded to the 16-bit format while the
    row sums stay fp32, P V accumulated in fp32, out = 16-bit(o * (1 / l)).  Exact exp2 / reciprocal (the kernel's
    approximations are within the error model's APPROX_REL)."""
    f32 = torch.float32
    x = qkv16.to(f32)
    n = x.shape[0]
    H = heads * 64
    out = torch.zeros(n, H, dtype=f32)
    keep = torch.as_tensor(keep).bool()
    bias = torch.where(keep, torch.tensor(0.0, dtype=f32), torch.tensor(-10000.0 * LOG2E, dtype=f32))
    sc = torch.tensor(LOG2E / 8.0, dtype=f32)
    for a in range(0, n, L):
        q = x[a:a + L, :H].view(-1, heads, 64).transpose(0, 1)
        k = x[a:a + L, H:2 * H].view(-1, heads, 64).transpose(0, 1)
        v = x[a:a + L, 2 * H:].view(-1, heads, 64).transpose(0, 1)
        s = q @ k.transpose(1, 2)                                        # fp32 accumulation
        t = (s.to(F64) * sc.to(F64) + bias[a:a + L].to(F64)).to(f32)    # one fma
        nb = max(1, L // 128)
        bw = min(L, 128)
        m_run = torch.full((heads, L, 1), -math.inf, dtype=f32)
        l = torch.zeros((heads, L, 1), dtype=f32)
        o = torch.zeros((heads, L, 64), dtype=f32)

        def exp_pass(tb, m_ref):
            pb = torch.exp2((tb - m_ref).to(f32))
            return pb, pb.to(dtype16(fmt)).to(f32)

        for j in range(nb):
            tb = t[..., j * bw:(j + 1) * bw]
            if j == 0:
                m_new = tb.max(-1, keepdim=True).values
                alpha = torch.zeros_like(m_new)
                pb, p16 = exp_pass(tb, m_new)
            else:
                m_new = m_run.clone()
                alpha = torch.ones_like(m_new)
                pb, p16 = exp_pass(tb, m_run)
                over = (tb - m_run).max(-1, keepdim=True).values
                warp_any = (over > 8.0).view(heads, L // 32, 32).any(-1, keepdim=True)
                redo = warp_any.expand(heads, L // 32, 32).reshape(heads, L, 1)
                m_red = torch.maximum(m_run, m_run + over)
                pr, pr16 = exp_pass(tb, m_red)
                m_new = torch.where(redo, m_red, m_new)
                alpha = torch.where(redo, torch.exp2(m_run - m_new), alpha)
                pb = torch.where(redo, pr, pb)
                p16 = torch.where(redo, pr16, p16)
            rsum = pb.sum(-1, keepdim=True)
            ob = p16 @ v[:, j * bw:(j + 1) * bw]
            o = o * alpha + ob
            l = l * alpha + rsum
            m_run = m_new
        y = (o * (1.0 / l)).to(dtype16(fmt)).to(f32)
        out[a:a + L] = y.transpose(0, 1).reshape(-1, H)
    return out


PLANT_COORDS = range(48, 64)   # head dims reserved for planted scores: zero in every q and k that is not planted


def random_qkv(n, heads, fmt, gen, sigma=1.1):
    """16-bit-valued qkv [n, 3 * 64 heads]: q, k ~ N(0, sigma^2) (scores ~ N(0, sigma^4) nats: sigma 1.1 gives the flat
    softmax of random weights), v ~ N(0, 1); the planting dims of q and k zeroed."""
    H = heads * 64
    x = torch.randn(n, 3 * H, generator=gen, dtype=F64)
    x[:, :2 * H] *= sigma
    x = x.view(n, 3, heads, 64)
    x[:, :2, :, PLANT_COORDS.start:] = 0.0
    return round16(x.view(n, 3 * H), fmt)


def plant(qkv, heads, fmt, row, head, key, ref_keys, delta, slot):
    """Give query `row` (head `head`) a score at `key` that exceeds its scores at `ref_keys` by `delta` log2 units,
    through planting dim `slot` (one per (row, key) pair in a head, so no other score changes).  Returns the planted
    excess actually reached after 16-bit rounding (log2 units)."""
    H = heads * 64
    h0 = head * 64
    c = h0 + PLANT_COORDS.start + slot
    q = qkv[row, h0:h0 + 64]
    base = (qkv[ref_keys, H + h0:H + h0 + 64] @ q).max().item() / 8.0
    s_key = (qkv[key, H + h0:H + h0 + 64] @ q).item() / 8.0
    a = 16.0
    qkv[row, c] = a
    want = base + delta / LOG2E
    qkv[key, H + c] = round16(torch.tensor((want - s_key) * 8.0 / a, dtype=F64), fmt)
    q = qkv[row, h0:h0 + 64]
    new = (qkv[key, H + h0:H + h0 + 64] @ q).item() / 8.0
    return (new - base) * LOG2E


# ------------------------------------------------------------------------------------------------
# LayerNorm and embeddings
# ------------------------------------------------------------------------------------------------
def layer_norm_ref(x, g, b, eps, unbiased=False, eps_outside=False):
    """fp64 LayerNorm (biased variance, eps inside the square root).  Perturbations: `unbiased` (H - 1 divisor),
    `eps_outside` ((x - mean) / (sqrt(var) + eps))."""
    x = x.to(F64)
    H = x.shape[-1]
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).sum(-1, keepdim=True) / (H - 1 if unbiased else H)
    den = (var.sqrt() + eps) if eps_outside else (var + eps).sqrt()
    z = (x - mu) / den
    return z * g.to(F64) + b.to(F64), z


def layer_norm_tol(x, z, y, g, b, out_fmt):
    """Error model of ln_rows_kernel / ln_rows_multi_kernel / ln_rows_packed_kernel / embed_ln_kernel, per element:
      mean      every input passes through at most D = H/32 + 5 fp32 additions (a lane's H/32 terms, then the 5-level
                shuffle tree): |d mean| <= (D + 1) 2^-24 sum|x| / H, which moves z by |d mean| * rstd
      variance  the same summation depth on (x - mean)^2 plus rsqrtf (2 ulp): relative (D + 6) 2^-24 + 2^-21 on z
      affine    fp32 (z g) + b: 2^-23 (|z g| + |b|)
      output    1/2 ulp16(|y| + delta) for a 16-bit output, nothing for fp32."""
    x = x.to(F64)
    H = x.shape[-1]
    D = H // 32 + 5
    xm = x - x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt((xm ** 2).mean(-1, keepdim=True) + 1e-30)
    dmean = (D + 1) * U32 * x.abs().sum(-1, keepdim=True) / H
    g = g.to(F64).abs()
    zg = z.abs() * g
    d = dmean * rstd * g + zg * ((D + 6) * U32 + APPROX_REL) + 2.0 ** -23 * (zg + b.to(F64).abs())
    if out_fmt is not None:
        d = d + 0.5 * ulp16(y.abs() + d, out_fmt)
    return d


def position_ids(ids: torch.Tensor, roberta: bool, pad_id: int) -> torch.Tensor:
    if roberta:
        m = (ids != pad_id).long()
        return torch.cumsum(m, dim=1) * m + pad_id
    return torch.arange(ids.shape[1]).unsqueeze(0).expand_as(ids)


def embed_ref(ids, word, pos, typ, g, b, eps, roberta, pad_id):
    """(word + pos) + type in fp32 (the kernel's association), then LayerNorm in fp64.  -> (x fp32, y, z)."""
    ids = torch.as_tensor(ids).long()
    x = (word.float()[ids] + pos.float()[position_ids(ids, roberta, pad_id)]) + typ.float()[0]
    y, z = layer_norm_ref(x, g, b, eps)
    return x, y, z


# ------------------------------------------------------------------------------------------------
# GELU forms of gemm_store.cuh, emulated in fp32
# ------------------------------------------------------------------------------------------------
def gelu_coefficients():
    """The polynomial coefficients of gelu_erf2 and gelu_logistic2, parsed from the kernel source."""
    src = (ROOT / "ance_b200" / "csrc" / "gemm_store.cuh").read_text()

    def body(name):
        m = re.search(r"void " + name + r"\(.*?\n}\n", src, re.S)
        assert m, name
        return m.group(0)

    num = r"pack2\(([-+0-9.eE]+)f, \1f\)"
    erf = [float(c) for c in re.findall(num, body("gelu_erf2"))]
    logi = [float(c) for c in re.findall(num, body("gelu_logistic2"))]
    return erf, logi


def _fma32(a, b, c):
    with np.errstate(over="ignore", invalid="ignore"):
        return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def gelu_erf2_emulate(x: np.ndarray, coef) -> np.ndarray:
    """gelu_erf2 in fp32: relu(x) - 0.5 |x| (1 + a1|x| + ... + a6|x|^6)^-16 with an exact reciprocal."""
    f = np.float32
    x = x.astype(f)
    ax = np.abs(x)
    c = [f(v) for v in coef]   # a6 .. a1 (1/sqrt(2) folded in), 1, then the 0.5 constants, in source order
    p = _fma32(np.full_like(x, c[0]), ax, np.full_like(x, c[1]))
    for v in c[2:7]:
        p = _fma32(p, ax, np.full_like(x, v))
    with np.errstate(over="ignore"):
        for _ in range(4):
            p = (p * p).astype(f)
        r = (f(1.0) / p).astype(f)
    relu = _fma32(ax, np.full_like(x, f(0.5)), (x * f(0.5)).astype(f))
    return _fma32((ax * f(-0.5)).astype(f), r, relu)


def gelu_logistic2_emulate(x: np.ndarray, coef) -> np.ndarray:
    """gelu_logistic2 in fp32: x / (1 + 2^(x (c4 t^4 + ... + c0))), t = x^2, exact exp2 and reciprocal."""
    f = np.float32
    x = x.astype(f)
    c = [f(v) for v in coef[:5]]
    with np.errstate(over="ignore", invalid="ignore"):
        t = (x * x).astype(f)
        p = _fma32(np.full_like(x, c[0]), t, np.full_like(x, c[1]))
        for v in c[2:5]:
            p = _fma32(p, t, np.full_like(x, v))
        g = (p * x).astype(f)
        e = np.exp2(g.astype(np.float64)).astype(f)
        d = _fma32(e, np.ones_like(x), np.ones_like(x))
        return (x * (f(1.0) / d).astype(f)).astype(f)


# ------------------------------------------------------------------------------------------------
# reporting
# ------------------------------------------------------------------------------------------------
WIDE_MIN_WAVES = 10   # kWideMinWaves of encoder.cu


def wide_tiles(M: int, N: int) -> int:
    """128 x 256 tiles of an [M, N] output."""
    return -(-M // 128) * -(-N // 256)


def wide_threshold(sm_count: int) -> int:
    """Fewest wide tiles for which linear() runs a call with a 16-bit output only, act 0 and no dropout on
    tc05_gemm_wide_kernel (encoder.cu linear(): kWideMinWaves waves of one tile per SM)."""
    return WIDE_MIN_WAVES * sm_count


def wide_slice_rows(N: int, threshold: int) -> int:
    """Most rows (a multiple of 128) of an [M, N] call that stays below the threshold: the 128 x 128 tile."""
    return (threshold - 1) // -(-N // 256) * 128


LINEAR_WIDE_PERTURBATIONS = ("bias n+1", "residual row+1", "residual row^64", "acc col^64", "acc row^8")


def linear_discrimination_blocked(out, A, W, bias, R, out_fmt, block_elems=1 << 23):
    """discrimination(out, linear_ref, linear_tol, perturbed) of an act-0 linear with a 16-bit output, computed over
    blocks of 128-aligned rows (at most ~block_elems outputs each) so that large M stays within a few GB of fp64.
    The perturbed references are the outputs of plausible bugs of a 128 x 256 tile on two 64-row warpgroups:
      bias n+1          bias of the next column
      residual row+1    residual of the next row (off-by-one pitch; the last row wraps to row 0)
      residual row^64   residual from the other warpgroup's 64-row half of the tile
      acc col^64        accumulator columns from the neighbouring 64-column slab
      acc row^8         accumulator rows r and r + 8 swapped (the two rows a thread holds in the wgmma fragment)
    A partner row or column past the matrix keeps its own value.  -> (max err / bound, {name: (fraction rejected,
    median margin, rows)}) as discrimination returns."""
    M, N = out.shape
    dev = out.device
    block = max(128, block_elems // N // 128 * 128)
    cols = torch.arange(N, device=dev)
    col_x = torch.where((cols ^ 64) < N, cols ^ 64, cols)
    w = W.to(F64)
    b = None if bias is None else bias.to(F64)
    names = [n for n in LINEAR_WIDE_PERTURBATIONS
             if (n.startswith("bias") and bias is not None) or (n.startswith("residual") and R is not None)
             or n.startswith("acc")]
    err, hit, margins = 0.0, {n: 0 for n in names}, {n: [] for n in names}
    for r0 in range(0, M, block):
        r1 = min(M, r0 + block)
        rows = torch.arange(r0, r1, device=dev)
        a = A[r0:r1].to(F64)
        acc = a @ w.T
        r = None if R is None else R[r0:r1].to(F64)

        def compose(acc_, b_, r_):
            x_ = acc_ if b_ is None else acc_ + b_
            return x_, (x_ if r_ is None else x_ + r_)

        x, y = compose(acc, b, r)
        tol = linear_tol(a, W, x, y, r, 0, out_fmt)
        o = out[r0:r1].to(F64)
        err = max(err, ((o - y).abs() / tol).max().item())
        for n in names:
            if n == "bias n+1":
                p = compose(acc, torch.roll(b, -1), r)[1]
            elif n == "residual row+1":
                p = compose(acc, b, R[(rows + 1) % M].to(F64))[1]
            elif n == "residual row^64":
                p = compose(acc, b, R[torch.where((rows ^ 64) < M, rows ^ 64, rows)].to(F64))[1]
            elif n == "acc col^64":
                p = compose(acc[:, col_x], b, r)[1]
            else:
                p = compose(acc[torch.where((rows ^ 8) < M, rows ^ 8, rows) - r0], b, r)[1]
            changed = ((p - y).abs() / tol).amax(-1) > 2.0
            d = ((o - p).abs() / tol).amax(-1)[changed]
            hit[n] += int((d > 1.0).sum())
            margins[n].append(d.cpu())
            del p
    rep = {}
    for n in names:
        d = torch.cat(margins[n])
        rep[n] = (hit[n] / d.numel() if d.numel() else float("nan"), float(d.median()) if d.numel() else float("nan"),
                  int(d.numel()))
    return err, rep


def discrimination(out, ref, tol, perturbed, changed_rows=None):
    """(max |out - ref| / tol, {name: rejection}) where rejection = (fraction of the rows the perturbation changes by
    more than 2 tol on which out lies outside tol of it, median over those rows of max |out - pert| / tol, rows)."""
    out = out.to(F64)
    err = ((out - ref).abs() / tol).max().item()
    rep = {}
    for name, pert in perturbed.items():
        d_ref = ((pert - ref).abs() / tol).amax(-1)
        rows = d_ref > 2.0 if changed_rows is None else (changed_rows & (d_ref > 2.0))
        r = ((out - pert).abs() / tol).amax(-1)[rows]
        rep[name] = (int((r > 1.0).sum()) / r.numel() if r.numel() else float("nan"),
                     float(r.median()) if r.numel() else float("nan"), int(r.numel()))
    return err, rep
