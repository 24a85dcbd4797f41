"""fp64 reference, fp32 emulation and written per-element bound for the attention backward of sequences of 256, 384 or
512 tokens (csrc/attn_bwd_long.cuh: ance_dbg_attention_backward_long, the launch ance_encoder_backward makes for L > 128).

The exact result is encoder_grad_refs.attention_bwd_ref: dQKV of sum(dO o softmax(Q K^T / 8 + mask) V) in fp64 from the
16-bit operands the kernel reads.  The kernel's arithmetic (what `emulate` restates in fp32 torch):

  s  = fmaf(q.k, c, kbias)        c = fp32(log2(e) / 8); q.k on the tensor cores in the storage format, fp32 accumulation
  dP = dO . bf16(v)               bf16 operands (v converted from fp16 storage; exact for bf16 storage)
  m, l, sum_j 2^(s - m) dP        online over the key blocks of 64: at a new maximum the running sums are rescaled by
                                  2^(m_old - m_new); l and the dP sum each take 16 terms per lane, 2 shuffle levels and one
                                  rescaling fma per block
  P  = 2^(s - m) (1 / l)          D = (sum_j 2^(s - m) dP) / l   (= sum_j P_ij dP_ij, the <= 128 kernel's rowsum)
  dS8 = P (dP - D) / 8            fp32, then rounded to bf16 for the two products
  dQ = bf16(dS8) bf16(K)          dK = bf16(dS8)^T bf16(Q)          dV = bf16(P)^T dO

Bound (u = 2^-24 the fp32 unit roundoff, ub = 2^-8 bf16's, uc = ub for fp16 storage and 0 for bf16; |.| elementwise
magnitudes of the exact operands, no cancellation assumed anywhere):

* Tensor-core accumulation.  The products of a k-step are exact; their sum and the accumulator are added with
  truncation, up to twice round-to-nearest's error per addition.  Over n terms: tc(n) = 2 (n + 2) u times sum |terms|.
* Score (log2 units): tc(64) |q||k| c  +  u |q.k c| (the fma's product, c's own rounding)  +  u |s|  +  u |s - m|
  (the subtraction before exp2f).  The natural-unit error is that over log2(e); a score error d gives P a relative error
  d_j + max_j d (the normaliser), so eps_P = 2 max_{j: P_ij > 0} d_ij + (24 + 6 nkb) u, nkb = L / 64: exp2f (2 ulp) of the
  term and of each rescaling factor, 1 / l and the product, and the 16 + 2 + 2 nkb roundings of l.  A masked key of a row
  with an unmasked one sits 14427 log2 units below the maximum: 2^(s - m) is 0 in fp32 and P is 0 in fp64, so only keys
  with P > 0 set the row's eps_P (as in the <= 128 bound).
* dP: (uc + tc(64)) |dO||v|^T = e_dP.
* D: sum_j P e_dP  +  (eps_P + (22 + 2 nkb) u) sum_j P |dO||v|^T: the propagated dP error, P's error and the roundings of
  the dP sum (as for l) and of the final division.
* dS8 before rounding: P (e_dP + e_D) + (eps_P + 3 u) P (|dP|~ + |D|~) over 8, with |dP|~ = |dO||v|^T and
  |D|~ = sum_j P |dP|~; its bf16 rounding adds ub times (the magnitude + that error).
* dQ = sum_j bf16(dS8) bf16(K): (e_dS8 + (uc + tc(L)) (|dS8|~ + e_dS8)) |k|; dK the same over the queries with |q|.
* dV = sum_i bf16(P) dO: ((eps_P + ub (1 + eps_P)) P + tc(L) P (1 + eps_P + ub))^T |dO|.

The perturbation `drop_rowsum` (dS = P o dP, the softmax Jacobian's rowsum dropped) must fall outside the bound.

`attention_stage` is encoder_layer_refs.attention_stage for L > 128: the layer-by-layer mirror's attention stage, whose
upstream gradient dO carries its own bound e, under this kernel's bound evaluated at |dO| + e plus the magnitude of the
linear map in dO applied to e.
"""
from __future__ import annotations

import math

import torch

from tests import encoder_grad_refs as G
from tests import encoder_layer_refs as LR

F64 = torch.float64
U32 = 2.0 ** -24
UB = 2.0 ** -8
LOG2E = math.log2(math.e)


def _tc(n):
    return 2.0 * (n + 2) * U32


def _bf(x):
    return x.to(torch.bfloat16).to(x.dtype)


def attention_bwd_long_ref(qkv, kbias_log2, dout, B, L, heads, drop_rowsum=False):
    """dQKV [B*L, 3H] fp64 (dout: [B*L, H], zero rows where there is no upstream gradient)."""
    return G.attention_bwd_ref(qkv, kbias_log2, dout, B, L, heads, drop_jacobian=drop_rowsum)


def attention_bwd_long_tol(qkv, kbias_log2, dout, B, L, heads, fmt):
    uc = UB if fmt == "fp16" else 0.0
    nkb = L // 64
    c = LOG2E / 8.0
    qa, ka, va = G._split(qkv.to(F64).abs(), B, L, heads)
    qs, ks, _ = G._split(qkv.to(F64), B, L, heads)
    doa = dout.to(F64).abs().reshape(B, L, heads, 64).transpose(1, 2)
    p = G.attention_probs(qkv, kbias_log2, B, L, heads)
    qk = qs @ ks.transpose(-1, -2)
    s = qk * c + kbias_log2.to(F64).reshape(B, 1, 1, L)
    m = s.amax(-1, keepdim=True)
    d_log2 = _tc(64) * (qa @ ka.transpose(-1, -2)) * c + U32 * (qk * c).abs() + U32 * s.abs() + U32 * (s - m).abs()
    eps_p = 2.0 * (d_log2 / LOG2E * (p > 0)).amax(-1, keepdim=True) + (24 + 6 * nkb) * U32
    adp = doa @ va.transpose(-1, -2)
    e_dp = (uc + _tc(64)) * adp
    pd = (p * adp).sum(-1, keepdim=True)
    e_d = (p * e_dp).sum(-1, keepdim=True) + (eps_p + (22 + 2 * nkb) * U32) * pd
    ads8 = p * (adp + pd) / 8.0
    e_pre = (p * (e_dp + e_d) / 8.0) + (eps_p + 3 * U32) * ads8
    e_ds8 = e_pre + UB * (ads8 + e_pre)
    gq = e_ds8 + (uc + _tc(L)) * (ads8 + e_ds8)
    tdq = gq @ ka
    tdk = gq.transpose(-1, -2) @ qa
    tdv = ((eps_p + UB * (1 + eps_p)) * p + _tc(L) * p * (1 + eps_p + UB)).transpose(-1, -2) @ doa
    return torch.cat([G._merge(tdq, B, L, heads), G._merge(tdk, B, L, heads), G._merge(tdv, B, L, heads)], dim=1) + 1e-30


def attention_stage(qkv, kbias_log2, dout, edout, B, L, heads, fmt):
    """(dQKV fp64, its bound) of the mirror's attention stage at L in {256, 384, 512} for operand format fmt."""
    ref = G.attention_bwd_ref(qkv, kbias_log2, dout, B, L, heads)
    tol = attention_bwd_long_tol(qkv, kbias_log2, dout.abs() + edout, B, L, heads, fmt)
    return ref, tol + LR._attention_abs(qkv, kbias_log2, edout, B, L, heads)


def emulate(qkv, kbias_log2, dout, B, L, heads, fmt, drop_rowsum=False):
    """The kernel's stated arithmetic in fp32 torch (see the module docstring); dout [B*L, H] bf16 values."""
    f32 = torch.float32
    q, k, v = G._split(qkv.to(f32), B, L, heads)
    do = dout.to(f32).reshape(B, L, heads, 64).transpose(1, 2)
    conv = _bf if fmt == "fp16" else (lambda x: x)
    c = torch.tensor(LOG2E / 8.0, dtype=f32)
    kb = kbias_log2.to(f32).reshape(B, 1, 1, L)
    s = (q @ k.transpose(-1, -2)) * c + kb
    dp = do @ conv(v).transpose(-1, -2)
    m = torch.full(s.shape[:-1], -math.inf, dtype=f32)
    l = torch.zeros_like(m)
    dn = torch.zeros_like(m)
    for j in range(0, L, 64):
        sb, db = s[..., j:j + 64], dp[..., j:j + 64]
        mn = torch.maximum(m, sb.amax(-1))
        a = torch.exp2(m - mn)
        e = torch.exp2(sb - mn[..., None])
        l = l * a + e.sum(-1)
        dn = dn * a + (e * db).sum(-1)
        m = mn
    inv = 1.0 / l
    D = dn / l
    p = torch.exp2(s - m[..., None]) * inv[..., None]
    ds8 = (p * dp if drop_rowsum else p * (dp - D[..., None])) * 0.125
    dq = _bf(ds8) @ conv(k)
    dk = _bf(ds8).transpose(-1, -2) @ conv(q)
    dv = _bf(p).transpose(-1, -2) @ do
    return torch.cat([G._merge(dq, B, L, heads), G._merge(dk, B, L, heads), G._merge(dv, B, L, heads)], dim=1)


LOG2_MASK = -10000.0 * LOG2E


def kbias(B, L, kinds, g):
    """kbias [B*L] fp32 (log2 units) with sequence b masked as kinds[b % len(kinds)]: "prefix" (a random length), "holed"
    (random holes, token 0 kept), "allpad" (every key masked) or "full"."""
    keep = torch.ones(B, L, dtype=torch.bool)
    for b in range(B):
        kind = kinds[b % len(kinds)]
        if kind == "prefix":
            keep[b, int(torch.randint(1, L + 1, (1,), generator=g)):] = False
        elif kind == "holed":
            keep[b] = torch.rand(L, generator=g) < 0.6
            keep[b, 0] = True
        elif kind == "allpad":
            keep[b] = False
    return torch.where(keep, 0.0, LOG2_MASK).reshape(-1).float()


def inputs(B, L, heads, fmt, kinds, seed, cls_only, late_max=False):
    """(qkv 16-bit [B*L, 3H], kbias, dout bf16 as the hook takes it, dout [B*L, H] with zeros where there is none).
    late_max: in head 0 of sequence 0 the queries and the keys of the last block share one direction w, so that every
    query's largest score (about |w|^2 / 8 = 8 against a spread of ~1.5 for the other keys) lies in the last key block
    only (sequence 0 should then be unmasked: kinds[0] = "full")."""
    g = torch.Generator().manual_seed(seed)
    H = heads * 64
    dt = torch.float16 if fmt == "fp16" else torch.bfloat16
    x = torch.randn(B * L, 3 * H, generator=g, dtype=F64) * 1.5
    if late_max:
        w = torch.randn(64, generator=g, dtype=F64)
        x[:L, :64] = w + 0.2 * torch.randn(L, 64, generator=g, dtype=F64)
        x[L - 64:L, H:H + 64] = w + 0.2 * torch.randn(64, 64, generator=g, dtype=F64)
    qkv = x.to(dt)
    kb = kbias(B, L, kinds, g)
    rows = B if cls_only else B * L
    d = torch.randn(rows, H, generator=g, dtype=F64).to(torch.bfloat16)
    full = torch.zeros(B * L, H, dtype=torch.bfloat16)
    if cls_only:
        full[::L] = d
    else:
        full = d
    return qkv, kb, d, full
