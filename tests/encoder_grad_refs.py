"""fp64 references for the encoder's backward kernels (csrc/encoder_bwd.cuh), each with a written per-element bound.

Every reference takes the operands the kernel reads (16-bit values widened exactly, fp32 where the kernel reads fp32) and
returns the exact result in fp64.  The bounds model the kernels' fp32 arithmetic, with u = 2^-24 the fp32 unit roundoff:

* attention_bwd: S and dP are 64-term fp32 dot products, P is rebuilt with exp2f and one division, dV / dQ / dK are L-term
  dot products.  A dot product of n terms is within gamma_n = n u of the exact one times the sum of |terms| (Higham 3.5).
  Writing |.| for elementwise magnitude, the bound propagates the magnitudes through the chain with no cancellation:
      |dS|~ = P o (|dP|~ + rowsum(P o |dP|~)),  |dP|~ = |dO| |V|^T
      err(dS) = gamma_70 |dS|~ + eps_P P o (|dP|~ + 2 rowsum(P o |dP|~))     (eps_P: relative error of P)
      dV: gamma_(L+2) P^T |dO| + (eps_P P)^T |dO|      dQ: (gamma_(L+2) |dS|~ + err(dS)) |K| / 8      dK: the same with Q
  eps_P = 2 max_j |dS_ij| + 8u per row, |dS_ij| <= gamma_64 |q_i| |k_j| / 8 + 2u |s_ij| / log2(e) the error of the
  natural-unit score (s_ij: the log2-unit score including the -10000 log2(e) key bias, which dominates on masked keys).
* ln_bwd: every row sum is H / 32 terms per lane in sequence, then 5 shuffle levels: n1 = H / 32 + 5 roundings deep.
  Worst case, to first order in u (|.|: the magnitudes of the exact quantities):
      mean:  abs error dm <= gamma_n1 mean|x|          rstd: relative error rr <= gamma_(n1+3) / 2 + 3u
      xhat:  abs error dxh <= rstd dm + |xhat| (rr + 2u)
      mean(g):  gamma_(n1+1) mean|g|                   mean(g xhat):  dm2 <= gamma_(n1+2) mean|g xhat| + mean(|g| dxh)
      dx = rstd (g - mean(g) - xhat mean(g xhat)):
          rstd [(rr + 4u) (|g| + mean|g| + |xhat| mean|g xhat|) + gamma_(n1+1) mean|g| + dxh mean|g xhat| + |xhat| dm2]
  The column sums run over n = rows / (8 x 264) per warp + 8 warps + 264 blocks + 2 terms: gamma_n sum |terms|, plus
  the xhat error carried through them (sum |dy| dxh) and, for the column sum of dx, the dx bound itself.
* gelu_bwd: Phi(u) + u phi(u) with erfcf and expf (<= 2 ulp each): 8 u (Phi + |u| phi) + 8 u.
* gemm (dgrad / wgrad on bf16 operands, fp32 accumulation): gamma_K |A| |B|^T, the operands being the bf16 values.
* embeddings: the scatter-add of n fp32 rows into one table row: gamma_n sum |dE rows|.

Perturbed references model plausible bugs: the softmax Jacobian's rowsum term dropped, dgamma / dbeta swapped, the tanh
GELU's derivative, the position gradient shifted by one row.  Each must fall outside the bound.
"""
from __future__ import annotations

import math

import torch

F64 = torch.float64
U32 = 2.0 ** -24


def _g(n):
    return n * U32


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def _split(qkv, B, L, heads):
    H = heads * 64
    q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
    f = lambda t: t.reshape(B, L, heads, 64).transpose(1, 2)   # [B, h, L, 64]
    return f(q), f(k), f(v)


def _merge(t, B, L, heads):
    return t.transpose(1, 2).reshape(B * L, heads * 64)


def attention_probs(qkv, kbias_log2, B, L, heads):
    """P [B, h, L, L] in fp64 from the kernel's inputs (kbias in log2 units, as the forward stores it)."""
    q, k, _ = _split(qkv.to(F64), B, L, heads)
    s = q @ k.transpose(-1, -2) / 8.0 + kbias_log2.to(F64).reshape(B, 1, 1, L) / math.log2(math.e)
    return torch.softmax(s, dim=-1)


def attention_bwd_ref(qkv, kbias_log2, dout, B, L, heads, drop_jacobian=False):
    """dQKV [B*L, 3H] fp64 of sum(dout o softmax(Q K^T / 8 + mask) V)."""
    q, k, v = _split(qkv.to(F64), B, L, heads)
    do = dout.to(F64).reshape(B, L, heads, 64).transpose(1, 2)
    p = attention_probs(qkv, kbias_log2, B, L, heads)
    dv = p.transpose(-1, -2) @ do
    dp = do @ v.transpose(-1, -2)
    ds = p * dp if drop_jacobian else p * (dp - (p * dp).sum(-1, keepdim=True))
    dq = ds @ k / 8.0
    dk = ds.transpose(-1, -2) @ q / 8.0
    return torch.cat([_merge(dq, B, L, heads), _merge(dk, B, L, heads), _merge(dv, B, L, heads)], dim=1)


def attention_bwd_tol(qkv, kbias_log2, dout, B, L, heads):
    q, k, v = _split(qkv.to(F64).abs(), B, L, heads)
    do = dout.to(F64).abs().reshape(B, L, heads, 64).transpose(1, 2)
    p = attention_probs(qkv, kbias_log2, B, L, heads)
    qs, ks, _ = _split(qkv.to(F64), B, L, heads)
    s_log2 = (qs @ ks.transpose(-1, -2)) * (math.log2(math.e) / 8.0) + kbias_log2.to(F64).reshape(B, 1, 1, L)
    # the score is formed in fp32 in log2 units beside the -10000 log2(e) key bias: its rounding, u |s|, is the larger term
    # on masked keys (all-padding rows)
    ds_err = _g(64) * (q @ k.transpose(-1, -2)) / 8.0 + 2 * U32 * s_log2.abs() / math.log2(math.e)
    eps_p = 2.0 * ds_err.amax(-1, keepdim=True) + 8 * U32
    adp = do @ v.transpose(-1, -2)
    pd = (p * adp).sum(-1, keepdim=True)
    ads = p * (adp + pd)                                          # |dS| with no cancellation
    eds = _g(70) * ads + eps_p * p * (adp + 2 * pd)               # error of dS: dP, rowsum, product; and P's own error
    tdv = _g(L + 2) * (p.transpose(-1, -2) @ do) + (eps_p * p).transpose(-1, -2) @ do
    tdq = (_g(L + 2) * ads + eds) @ k / 8.0
    tdk = (_g(L + 2) * ads + eds).transpose(-1, -2) @ q / 8.0
    return torch.cat([_merge(tdq, B, L, heads), _merge(tdk, B, L, heads), _merge(tdv, B, L, heads)], dim=1) + 1e-30


# ------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------
def ln_bwd_ref(x, gamma, eps, dy, swap_gb=False):
    """(dx, dgamma, dbeta, dsum = column sum of dx) in fp64."""
    x, gamma, dy = x.to(F64), gamma.to(F64), dy.to(F64)
    mean = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + eps)
    xh = (x - mean) * rstd
    g = dy * gamma
    dx = rstd * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    dgamma, dbeta = (dy * xh).sum(0), dy.sum(0)
    if swap_gb:
        dgamma, dbeta = dbeta, dgamma
    return dx, dgamma, dbeta, dx.sum(0)


def ln_bwd_tol(x, gamma, eps, dy):
    x, gamma, dy = x.to(F64), gamma.to(F64), dy.to(F64)
    rows, H = x.shape
    n1 = H // 32 + 5
    mean = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + eps)
    xh = ((x - mean) * rstd).abs()
    g = (dy * gamma).abs()
    dm = _g(n1) * x.abs().mean(-1, keepdim=True)
    rr = _g(n1 + 3) / 2 + 3 * U32
    dxh = rstd * dm + xh * (rr + 2 * U32)
    m1a, m2a = g.mean(-1, keepdim=True), (g * xh).mean(-1, keepdim=True)
    dm2 = _g(n1 + 2) * m2a + (g * dxh).mean(-1, keepdim=True)
    dx_abs = rstd * (g + m1a + xh * m2a)
    tdx = (rr + 4 * U32) * dx_abs + rstd * (_g(n1 + 1) * m1a + dxh * m2a + xh * dm2) + 1e-30
    n = -(-rows // (8 * 264)) + 8 + 264 + 2
    tg = _g(n) * (dy.abs() * xh).sum(0) + (dy.abs() * dxh).sum(0) + 1e-30
    tb = _g(n) * dy.abs().sum(0) + 1e-30
    ts = _g(n) * dx_abs.sum(0) + tdx.sum(0)
    return tdx, tg, tb, ts


# ------------------------------------------------------------------------------------------------
# GELU
# ------------------------------------------------------------------------------------------------
def gelu_bwd_ref(u, tanh_form=False):
    u = u.to(F64)
    if tanh_form:
        c = math.sqrt(2.0 / math.pi)
        t = torch.tanh(c * (u + 0.044715 * u ** 3))
        return 0.5 * (1 + t) + 0.5 * u * (1 - t * t) * c * (1 + 3 * 0.044715 * u * u)
    phi = torch.exp(-0.5 * u * u) / math.sqrt(2 * math.pi)
    Phi = 0.5 * torch.erfc(-u / math.sqrt(2.0))
    return Phi + u * phi


def gelu_bwd_tol(u):
    u = u.to(F64)
    phi = torch.exp(-0.5 * u * u) / math.sqrt(2 * math.pi)
    Phi = 0.5 * torch.erfc(-u / math.sqrt(2.0))
    return 8 * U32 * (Phi + u.abs() * phi) + 8 * U32


# ------------------------------------------------------------------------------------------------
# GEMM (dgrad / wgrad) and embeddings
# ------------------------------------------------------------------------------------------------
def gemm_ref(A, B):
    """A [M, K] @ B [K, N] in fp64 (A, B: the bf16 operand values)."""
    return A.to(F64) @ B.to(F64)


def gemm_tol(A, B):
    return _g(A.shape[1] + 2) * (A.to(F64).abs() @ B.to(F64).abs()) + 1e-30


def position_ids(ids, pad_id, roberta=True):
    if roberta:
        m = (ids != pad_id).long()
        return torch.cumsum(m, dim=1) * m + pad_id
    return torch.arange(ids.shape[1]).unsqueeze(0).expand_as(ids)


def embedding_grads_ref(ids, dE, vocab, max_pos, pad_id, roberta=True, pos_shift=0):
    """(d word [vocab, H], d pos [max_pos, H]) of the embedding sum (word[id] + pos[p]) with gradient dE [B*L, H]; the
    padding rows (word pad_id; position pad_id for RoBERTa) get none, as nn.Embedding(padding_idx=...) gives them."""
    H = dE.shape[1]
    ids = ids.long()
    pos = (position_ids(ids, pad_id, roberta) + pos_shift).clamp(0, max_pos - 1).reshape(-1)
    idf = ids.reshape(-1)
    dE = dE.to(F64)
    dw = torch.zeros(vocab, H, dtype=F64).index_add_(0, idf, dE)
    dp = torch.zeros(max_pos, H, dtype=F64).index_add_(0, pos, dE)
    dw[pad_id] = 0
    if roberta:
        dp[pad_id] = 0
    return dw, dp


def embedding_grads_tol(ids, dE, vocab, max_pos, pad_id, roberta=True):
    ids = ids.long()
    a = dE.to(F64).abs()
    cnt_w = torch.bincount(ids.reshape(-1), minlength=vocab).to(F64)
    pos = position_ids(ids, pad_id, roberta).reshape(-1)
    cnt_p = torch.bincount(pos, minlength=max_pos).to(F64)
    sw = torch.zeros(vocab, a.shape[1], dtype=F64).index_add_(0, ids.reshape(-1), a)
    sp = torch.zeros(max_pos, a.shape[1], dtype=F64).index_add_(0, pos, a)
    return (cnt_w[:, None] + 1) * U32 * sw + 1e-30, (cnt_p[:, None] + 1) * U32 * sp + 1e-30


def discrimination(out, ref, tol, perturbed: dict):
    """(max |out - ref| / tol, {name: fraction of the changed elements' rows ... }) — a perturbed reference is rejected
    when the kernel's output lies outside the bound around it somewhere."""
    out, ref, tol = out.to(F64), ref.to(F64), tol.to(F64)
    err = float(((out - ref).abs() / tol).max())
    rep = {k: float(((out - p.to(F64)).abs() / tol).max()) for k, p in perturbed.items()}
    return err, rep
