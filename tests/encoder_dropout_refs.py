"""Dropout of the training forward / backward: the numpy generator, mask builders and fp64 mirrors with masks.

The scheme (DESIGN.md §4.1, csrc/dropout.cuh), restated bit for bit:
  Philox4x32-10, key (seed & 0xffffffff, seed >> 32).
  hidden sites (0 embeddings, 2 attention output, 3 FFN output), token t = b L + i, column n:
      counter (n >> 3, t, 0, 4 layer + site), 16 bits: word (n >> 1) & 3, half n & 1 (half 0 = low bits)
  attention probabilities (site 1), sequence b, head h, query i, key j:
      counter (4 (j >> 5) + ((j >> 1) & 3), i, b heads + h, 4 layer + 1), 16 bits: word (j >> 3) & 3, half j & 1
  keep  <=>  u16 >= thr,  thr = min(round(p 2^16), 65535);  p_eff = thr / 2^16;  kept values scaled by 1 / (1 - p_eff).

The fp64 mirrors of the attention and hidden-site backward take the masks (0 / 1 arrays) and the scale explicitly, with
flags for the mistakes a test must be able to tell apart; masked_hidden_states is the fp32 oracle forward with the same
masks, for end-to-end gradients through torch.autograd.
"""
from __future__ import annotations

import functools

import numpy as np

M0, M1 = np.uint32(0xD2511F53), np.uint32(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
SITE_EMBED, SITE_ATTN, SITE_ATTN_OUT, SITE_FFN_OUT = 0, 1, 2, 3


def _mulhilo(a, b):
    p = a.astype(np.uint64) * np.uint64(b)
    return (p >> np.uint64(32)).astype(np.uint32), (p & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def philox(seed: int, c0, c1, c2, c3) -> np.ndarray:
    """Philox4x32-10 of the counters (broadcast uint32 arrays) under the 64-bit key `seed` -> uint32 [..., 4]."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint32) for c in np.broadcast_arrays(c0, c1, c2, c3))
    k0, k1 = np.uint32(seed & 0xFFFFFFFF), np.uint32((seed >> 32) & 0xFFFFFFFF)
    with np.errstate(over="ignore"):
        for r in range(10):
            if r:
                k0, k1 = np.uint32(k0 + W0), np.uint32(k1 + W1)
            hi0, lo0 = _mulhilo(c0, M0)
            hi1, lo1 = _mulhilo(c2, M1)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    return np.stack([c0, c1, c2, c3], axis=-1)


def philox_key(k0: int, k1: int, ctr) -> np.ndarray:
    """Philox4x32-10 with an explicit (k0, k1) key and one 4-word counter (Random123's known-answer form)."""
    return philox(int(k0) | (int(k1) << 32), *[np.uint32(c) for c in ctr])


def dbg_bits(seed: int, stream_word: int, first: int, n: int) -> np.ndarray:
    """What ance_dbg_dropout_bits writes: call i has the counter (lo32(first + i), hi32(first + i), lo32(stream_word),
    hi32(stream_word)); -> uint32 [4 n]."""
    x = np.uint64(first) + np.arange(n, dtype=np.uint64)
    lo = (x & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    hi = (x >> np.uint64(32)).astype(np.uint32)
    return philox(seed, lo, hi, np.uint32(stream_word & 0xFFFFFFFF), np.uint32(stream_word >> 32)).reshape(-1)


def threshold(p: float) -> int:
    return min(int(np.rint(p * 65536.0)), 65535)


def p_eff(p: float) -> float:
    return threshold(p) / 65536.0


def scale(p: float) -> float:
    """The scale of kept values as the library computes it (fp32)."""
    return float(np.float32(1.0) / np.float32(1.0 - p_eff(p)))


def stream(site: int, layer: int) -> int:
    return 4 * layer + site


def _half16(w: np.ndarray, word: np.ndarray, half: np.ndarray) -> np.ndarray:
    v = np.take_along_axis(w, word[..., None].astype(np.int64), axis=-1)[..., 0]
    return (v >> (16 * half).astype(np.uint32)) & np.uint32(0xFFFF)


def hidden_mask(seed: int, site: int, layer: int, tokens, H: int, p: float) -> np.ndarray:
    """0 / 1 mask [len(tokens), H] of a hidden site for the given token indices t = b L + i."""
    t = np.asarray(tokens, dtype=np.uint32)[:, None]
    n = np.arange(H, dtype=np.uint32)
    w = philox(seed, np.arange(H // 8, dtype=np.uint32)[None, :], t, 0, stream(site, layer))   # one call per 8 columns
    u = (w[:, n >> 3, (n >> 1) & 3] >> (16 * (n & 1))) & np.uint32(0xFFFF)
    return (u >= threshold(p)).astype(np.float64)


def attn_mask(seed: int, layer: int, b: int, h: int, heads: int, L: int, p: float, queries=None) -> np.ndarray:
    """0 / 1 mask [len(queries), L] of the attention probabilities of (sequence b, head h): rows = queries i, columns =
    keys j."""
    i = np.arange(L, dtype=np.uint32)[:, None] if queries is None else np.asarray(queries, dtype=np.uint32)[:, None]
    j = np.arange(L, dtype=np.uint32)
    nc = 4 * ((L + 31) // 32)
    w = philox(seed, np.arange(nc, dtype=np.uint32)[None, :], i, b * heads + h, stream(SITE_ATTN, layer))   # one per 8 keys
    u = (w[:, 4 * (j >> 5) + ((j >> 1) & 3), (j >> 3) & 3] >> (16 * (j & 1))) & np.uint32(0xFFFF)
    return (u >= threshold(p)).astype(np.float64)


@functools.lru_cache(maxsize=64)
def _attn_masks(seed: int, layer: int, B: int, heads: int, L: int, p: float) -> np.ndarray:
    m = np.stack([np.stack([attn_mask(seed, layer, b, h, heads, L, p) for h in range(heads)]) for b in range(B)])
    m.flags.writeable = False
    return m


def attn_masks(seed: int, layer: int, B: int, heads: int, L: int, p: float) -> np.ndarray:
    """[B, heads, L, L] 0 / 1 (cached: read-only)."""
    return _attn_masks(int(seed), int(layer), int(B), int(heads), int(L), float(p))


# ------------------------------------------------------------------------------------------------------------------
# fp64 mirrors with masks
# ------------------------------------------------------------------------------------------------------------------
def attention_fwd(q, k, v, kbias_nat, m, s):
    """ctx = (m o softmax(q k^T / 8 + kbias) s) v for one (sequence, head): q, k, v [L, 64], kbias_nat [L] (natural
    units), m [Lq, L] 0/1 (Lq rows of q).  Returns (ctx, P)."""
    S = q @ k.T / 8.0 + kbias_nat[None, :]
    S = S - S.max(axis=1, keepdims=True)
    P = np.exp(S)
    P /= P.sum(axis=1, keepdims=True)
    return (P * m * s) @ v, P


def attention_bwd(q, k, v, kbias_nat, do, m, s, *, mask_bwd=True, scale_bwd=True, d_from_unmasked=False,
                  transpose_mask=False):
    """dq, dk, dv of one (sequence, head) with the dropout mask m [L, L] and scale s, in fp64.  The keyword flags are
    the perturbations the bounds must reject: mask not applied, 1 / (1 - p) missing, D from the unmasked dO V^T, the
    mask indexed (j, i)."""
    S = q @ k.T / 8.0 + kbias_nat[None, :]
    S = S - S.max(axis=1, keepdims=True)
    P = np.exp(S)
    P /= P.sum(axis=1, keepdims=True)
    mm = m.T if transpose_mask else m
    mb = mm if mask_bwd else np.ones_like(mm)
    sb = s if scale_bwd else 1.0
    Pt = P * mb * sb
    dv = Pt.T @ do
    dPraw = do @ v.T
    dP = dPraw * mb * sb
    D = (P * (dPraw if d_from_unmasked else dP)).sum(axis=1, keepdims=True)
    dS = P * (dP - D) / 8.0
    return dS @ k, dS.T @ q, dv


def layer_norm_bwd(x, g, dy, eps):
    mu = x.mean(axis=1, keepdims=True)
    var = ((x - mu) ** 2).mean(axis=1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + eps)
    xh = (x - mu) * rstd
    gg = dy * g[None, :]
    dx = rstd * (gg - gg.mean(axis=1, keepdims=True) - xh * (gg * xh).mean(axis=1, keepdims=True))
    return dx, (dy * xh).sum(0), dy.sum(0)


def dropout_linear_bwd(dT, m, s, x, w, *, mask_residual=False, bias_unmasked=False, mask_bwd=True, scale_bwd=True):
    """Backward of T = m o (x W^T + b) s + R at the LayerNorm input gradient dT: returns (d_branch_input, dW, db,
    d_residual).  Flags: the perturbations the bounds must reject."""
    mb = m if mask_bwd else np.ones_like(m)
    sb = s if scale_bwd else 1.0
    dTm = dT * mb * sb
    dres = dTm if mask_residual else dT
    db = (dT if bias_unmasked else dTm).sum(0)
    return dTm @ w, dTm.T @ x, db, dres


# ------------------------------------------------------------------------------------------------------------------
# the fp32 oracle with the same masks (a restatement of oracle/encoder_oracle.py's forward, dropout added at the four
# sites of HF transformers 2.3.0 in training mode)
# ------------------------------------------------------------------------------------------------------------------
def masked_hidden_states(o, ids, mask, seed: int, p_hidden: float, p_attn: float):
    """Last-layer hidden states [B, L, H] of the EncoderOracle `o` (its sd may hold autograd leaves) with the library's
    dropout masks of `seed`.  fp32 torch on o's device."""
    import math

    import torch
    import torch.nn.functional as F

    dev = o.device
    ids = ids.to(dev).long()
    mask = torch.as_tensor(mask).to(dev)
    B, L = ids.shape
    x = (o.w("embeddings.word_embeddings.weight")[ids] + o.w("embeddings.position_embeddings.weight")[o.position_ids(ids)]
         + o.w("embeddings.token_type_embeddings.weight")[0])
    x = F.layer_norm(x, (x.shape[-1],), o.w("embeddings.LayerNorm.weight"), o.w("embeddings.LayerNorm.bias"), o.eps)
    H = x.shape[-1]
    dh = H // o.heads
    tokens = np.arange(B * L)

    def hmask(site, layer):
        if p_hidden == 0:
            return 1.0
        m = hidden_mask(seed, site, layer, tokens, H, p_hidden) * scale(p_hidden)
        return torch.tensor(m, dtype=torch.float32, device=dev).view(B, L, H)

    x = x * hmask(SITE_EMBED, 0)
    ext = (1.0 - mask.float())[:, None, None, :] * -10000.0
    for l in range(o.n_layer):
        lp = f"encoder.layer.{l}."
        q = F.linear(x, o.w(lp + "attention.self.query.weight"), o.w(lp + "attention.self.query.bias"))
        k = F.linear(x, o.w(lp + "attention.self.key.weight"), o.w(lp + "attention.self.key.bias"))
        v = F.linear(x, o.w(lp + "attention.self.value.weight"), o.w(lp + "attention.self.value.bias"))
        q, k, v = (t.view(B, L, o.heads, dh).transpose(1, 2) for t in (q, k, v))
        pr = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(dh) + ext, dim=-1)
        if p_attn > 0:
            am = attn_masks(seed, l, B, o.heads, L, p_attn) * scale(p_attn)
            pr = pr * torch.tensor(am, dtype=torch.float32, device=dev)
        a = (pr @ v).transpose(1, 2).reshape(B, L, H)
        a = F.linear(a, o.w(lp + "attention.output.dense.weight"), o.w(lp + "attention.output.dense.bias"))
        x = F.layer_norm(a * hmask(SITE_ATTN_OUT, l) + x, (H,), o.w(lp + "attention.output.LayerNorm.weight"),
                         o.w(lp + "attention.output.LayerNorm.bias"), o.eps)
        h = F.gelu(F.linear(x, o.w(lp + "intermediate.dense.weight"), o.w(lp + "intermediate.dense.bias")))
        h = F.linear(h, o.w(lp + "output.dense.weight"), o.w(lp + "output.dense.bias"))
        x = F.layer_norm(h * hmask(SITE_FFN_OUT, l) + x, (H,), o.w(lp + "output.LayerNorm.weight"),
                         o.w(lp + "output.LayerNorm.bias"), o.eps)
    return x


# ------------------------------------------------------------------------------------------------------------------
# the layer-by-layer mirror (tests/encoder_layer_refs.py) with masks
# ------------------------------------------------------------------------------------------------------------------
# Perturbations of the backward's dropout rules; the GPU test asserts that the bound rejects each of them.
PERTURBATIONS = ("no_mask_bwd", "no_scale_bwd", "residual_masked", "bias_unmasked", "d_unmasked", "mask_transposed")
_U32 = 2.0 ** -24


def masked_attention_bwd_ref(qkv, kbias_log2, dout, B, L, heads, am, s, perturb=None):
    """dQKV [B L, 3H] fp64 of the attention with dropout mask am [B, heads, L, L] (0 / 1) and scale s:
    P~ = m o P s, dV = P~^T dO, dP = m o (dO V^T) s, D = sum_j P dP, dS = P o (dP - D)."""
    import torch

    from tests import encoder_grad_refs as G
    f64 = torch.float64
    q, k, v = G._split(qkv.to(f64), B, L, heads)
    do = dout.to(f64).reshape(B, L, heads, 64).transpose(1, 2)
    p = G.attention_probs(qkv, kbias_log2, B, L, heads)
    m = am.transpose(-1, -2) if perturb == "mask_transposed" else am
    if perturb == "no_mask_bwd":
        m = torch.ones_like(m)
    sb = 1.0 if perturb == "no_scale_bwd" else s
    dv = (p * m * sb).transpose(-1, -2) @ do
    dpr = do @ v.transpose(-1, -2)
    dp = dpr * m * sb
    D = (p * (dpr if perturb == "d_unmasked" else dp)).sum(-1, keepdim=True)
    ds = p * (dp - D)
    return torch.cat([G._merge(ds @ k / 8.0, B, L, heads), G._merge(ds.transpose(-1, -2) @ q / 8.0, B, L, heads),
                      G._merge(dv, B, L, heads)], dim=1)


def masked_attention_stage(qkv, kbias_log2, dout, edout, B, L, heads, fmt, am, s, perturb=None):
    """(dQKV, bound) of the masked attention stage.  Every magnitude the dropout backward forms (P~ <= s P, |dP| <= s
    |dO||V|^T, |D| <= s sum_j P |dO||V|^T, hence |dS| and the products) is at most s times the one the unmasked bound is
    built from, and the bounds are monotone in those magnitudes; the two extra fp32 products by s add 2 u relative.  So
    the unmasked stage's bound (encoder_layer_refs / encoder_grad_long_refs at |dO| + e) times s (1 + 4 u) bounds it."""
    from tests import encoder_grad_long_refs as R
    from tests import encoder_layer_refs as LR
    ref = masked_attention_bwd_ref(qkv, kbias_log2, dout, B, L, heads, am, s, perturb)
    if L <= 128:
        tol = LR.attention_stage(qkv, kbias_log2, dout, edout, B, L, heads)[1]
    else:
        tol = R.attention_stage(qkv, kbias_log2, dout, edout, B, L, heads, fmt)[1]
    return ref, tol * s * (1 + 4 * _U32)


def _site_bwd(dT, eT, m, s, perturb):
    """The branch gradient m o dT s of a hidden site with its bound (one fp32 product by s in mask_rows)."""
    mm = 1.0 if perturb == "no_mask_bwd" else m
    sb = 1.0 if perturb == "no_scale_bwd" else s
    a = dT * mm * sb
    return a, eT * mm * sb + _U32 * a.abs()


def packed_hidden_mask(seed: int, site: int, layer: int, row_tok, H: int, p: float, perturb=None) -> np.ndarray:
    """0 / 1 mask [M, H] of a hidden site over the rows of a packed plan: row r has token row_tok[r]'s mask (a row of no
    sequence, row_tok -1, gets 0: its gradient is 0 whatever the mask).  perturb "hidden_mask_by_row" keys the mask by
    the row index r instead."""
    tok = np.asarray(row_tok, dtype=np.int64)
    keys = np.arange(len(tok)) if perturb == "hidden_mask_by_row" else np.maximum(tok, 0)
    return hidden_mask(seed, site, layer, keys, H, p) * (tok >= 0)[:, None]


def packed_attn_masks(seed: int, layer: int, B: int, heads: int, L: int, p: float, seq_row0=None, perturb=None):
    """[B, heads, L, L] 0 / 1: the dense batch's masks (attn_masks), which a packed plan uses too.  perturb
    "attn_mask_from_tile": the (query, key) counters of sequence b start at its first row's offset in its tile,
    seq_row0[b] mod 128, instead of 0."""
    if perturb != "attn_mask_from_tile":
        return attn_masks(seed, layer, B, heads, L, p)
    out = np.empty((B, heads, L, L))
    for b in range(B):
        o = int(seq_row0[b]) % 128
        for h in range(heads):
            out[b, h] = attn_mask(seed, layer, b, h, heads, L + o, p, queries=np.arange(L) + o)[:, o:o + L]
    return out


def masked_layer_bwd_ref(act, kbias, w, dy, B, L, heads, last, eps, fmt, hm_out, hm_ffn, am, s, perturb=None,
                         plan=None, exact=False):
    """encoder_layer_refs.layer_bwd_ref with dropout: hm_out / hm_ffn the 0 / 1 masks [Mr, H] of sites 2 / 3 (the CLS
    rows' masks in the pruned last layer), am [B, heads, L, L] site 1's, s the scale.  The residual gets the LayerNorm's
    dT; the bias gradient, wgrad and dgrad get m o dT s.  plan: a packed plan, as in layer_bwd_ref (the masks then those
    of packed_hidden_mask / packed_attn_masks); exact: no bf16 conversions, as in layer_bwd_ref."""
    import torch

    from tests import encoder_layer_refs as LR
    cv = (lambda t: t.to(torch.float64)) if exact else LR.to_bf16
    F64 = torch.float64
    dy = dy.to(F64)
    M = B * L if plan is None else plan[3]
    g, t = {}, {}
    (dT, g["ln2_g"], g["ln2_b"], bu), (eT, t["ln2_g"], t["ln2_b"], tu) = LR.ln_stage(act["t2"], w["ln2_g"], eps, dy,
                                                                                     torch.zeros_like(dy))
    dTm, eTm = _site_bwd(dT, eT, hm_ffn, s, perturb)
    g["ff2_b"], t["ff2_b"] = (bu, tu) if perturb == "bias_unmasked" else LR._colsum(dTm, eTm)
    A, eA = LR._rnd(dTm, eTm, exact)
    g["ff2_w"], t["ff2_w"] = LR._mm(A.t(), eA.t(), cv(act["ff"]))
    dF, eF = LR._mm(A, eA, cv(w["w2"]))
    G = LR.G
    d = G.gelu_bwd_ref(act["u"])
    td = G.gelu_bwd_tol(act["u"])
    dU = dF * d
    eU = eF * (d.abs() + td) + dF.abs() * td + _U32 * (dF.abs() + eF) * (d.abs() + td)
    g["ff1_b"], t["ff1_b"] = LR._colsum(dU, eU)
    A, eA = LR._rnd(dU, eU, exact)
    g["ff1_w"], t["ff1_w"] = LR._mm(A.t(), eA.t(), cv(act["x1"]))
    dX1, eX1 = LR._mm(A, eA, cv(w["w1"]))
    dX1, eX1 = LR._add(dX1, eX1, *((dTm, eTm) if perturb == "residual_masked" else (dT, eT)))
    (dT1, g["ln1_g"], g["ln1_b"], bu), (eT1, t["ln1_g"], t["ln1_b"], tu) = LR.ln_stage(act["t1"], w["ln1_g"], eps, dX1, eX1)
    dT1m, eT1m = _site_bwd(dT1, eT1, hm_out, s, perturb)
    g["ao_b"], t["ao_b"] = (bu, tu) if perturb == "bias_unmasked" else LR._colsum(dT1m, eT1m)
    A, eA = LR._rnd(dT1m, eT1m, exact)
    ctx = LR.last_ctx(act, B, L, plan, perturb) if last else act["ctx"]
    g["ao_w"], t["ao_w"] = LR._mm(A.t(), eA.t(), cv(ctx))
    dC, eC = LR._rnd(*LR._mm(A, eA, cv(w["wo"])), exact)
    H = dC.shape[1]
    if last:
        dO, eO = torch.zeros(M, H, dtype=F64, device=dC.device), torch.zeros(M, H, dtype=F64, device=dC.device)
        rows = slice(None, None, L) if plan is None else plan[0].to(dC.device).long()
        dO[rows], eO[rows] = dC, eC
    else:
        dO, eO = dC, eC
    ap = perturb if perturb in ("no_mask_bwd", "no_scale_bwd", "d_unmasked", "mask_transposed") else None
    stage = lambda q, kb, do, edo, B_, L_, h: masked_attention_stage(q, kb, do, edo, B_, L_, h, fmt, am, s, ap)
    if plan is None:
        dA, eA3 = stage(act["qkv"], kbias, dO, eO, B, L, heads)
    else:
        dA, eA3 = LR.packed_attention(stage, act["qkv"], kbias, dO, eO, B, L, heads, plan)
    bq, tq = LR._colsum(dA, eA3)
    g["q_b"], g["k_b"], g["v_b"] = bq[:H], bq[H:2 * H], bq[2 * H:]
    t["q_b"], t["k_b"], t["v_b"] = tq[:H], tq[H:2 * H], tq[2 * H:]
    A, eA = LR._rnd(dA, eA3, exact)
    xt = cv(act["x_in"])
    for i, n in enumerate(("q_w", "k_w", "v_w")):
        sl = slice(i * H, (i + 1) * H)
        g[n], t[n] = LR._mm(A[:, sl].t(), eA[:, sl].t(), xt)
    dX, eX = LR._mm(A, eA, cv(w["wqkv"]))
    dX, eX = dX.clone(), eX.clone()
    res, eres = (dT1m, eT1m) if perturb == "residual_masked" else (dT1, eT1)
    if last and plan is not None:
        rows, keep = LR.cls_rows(B, L, M, plan, perturb, dX.device)
        res, eres = res[keep], eres[keep]
    else:
        rows = slice(None, None, L) if last else slice(None)
    dX[rows], eX[rows] = LR._add(dX[rows], eX[rows], res, eres)
    g["x_in"], t["x_in"] = dX, eX
    return g, t


def masked_autograd_grads(sd, batches, seeds, objective, p_hidden, p_attn, fmt=None, n_layer=12, heads=12, pad=1,
                          eps=1e-5):
    """tests/test_gpu_encoder_backward_layers._autograd_grads (fp32 autograd of RoBERTa + head, TF32 off; fmt: every
    value the encoder stores in 16 bits rounded to it, gradient passed straight through) with the library's masks of
    seeds[i] for batches[i]."""
    import torch
    import torch.nn.functional as Fn

    from tests import encoder_grad_refs as G
    dt = {"fp16": torch.float16, "bf16": torch.bfloat16}
    r = (lambda t: t) if fmt is None else (lambda t: t + (t.to(dt[fmt]).float() - t).detach())
    leaves = {k: v.detach().float().cuda().requires_grad_(True) for k, v in sd.items()}
    w = lambda n: leaves["roberta." + n]
    ln = lambda x, p: Fn.layer_norm(x, (x.shape[-1],), w(p + ".weight"), w(p + ".bias"), eps)
    s_h, s_a = np.float32(scale(p_hidden)), np.float32(scale(p_attn))

    def emb(ids, mask, seed):
        ids, mask = ids.cuda(), mask.cuda()
        B, L = ids.shape
        H = w("embeddings.word_embeddings.weight").shape[1]
        hm = lambda site, l: torch.tensor(hidden_mask(seed, site, l, np.arange(B * L), H, p_hidden) * s_h,
                                          dtype=torch.float32, device="cuda").view(B, L, H)
        pos = G.position_ids(ids.cpu(), pad).cuda()
        x = (w("embeddings.word_embeddings.weight")[ids] + w("embeddings.position_embeddings.weight")[pos]) + \
            w("embeddings.token_type_embeddings.weight")[0]
        x = r(ln(x, "embeddings.LayerNorm") * hm(SITE_EMBED, 0))
        ext = (1.0 - mask.float())[:, None, None, :] * -10000.0
        for l in range(n_layer):
            p = f"encoder.layer.{l}."
            lin = lambda t, n: Fn.linear(t, r(w(p + n + ".weight")), w(p + n + ".bias"))
            hd = lambda t: r(t).view(B, L, heads, 64).transpose(1, 2)
            q, k, v = hd(lin(x, "attention.self.query")), hd(lin(x, "attention.self.key")), hd(lin(x, "attention.self.value"))
            am = torch.tensor(attn_masks(seed, l, B, heads, L, p_attn) * s_a, dtype=torch.float32, device="cuda")
            a = r(((torch.softmax(q @ k.transpose(-1, -2) / 8.0 + ext, dim=-1) * am) @ v).transpose(1, 2).reshape(B, L, -1))
            x1 = r(ln(r(lin(a, "attention.output.dense") * hm(SITE_ATTN_OUT, l) + x), p + "attention.output.LayerNorm"))
            ff = r(Fn.gelu(lin(x1, "intermediate.dense")))
            x = r(ln(r(lin(ff, "output.dense") * hm(SITE_FFN_OUT, l) + x1), p + "output.LayerNorm"))
        hin = Fn.linear(x[:, 0], r(leaves["embeddingHead.weight"]), leaves["embeddingHead.bias"])
        return Fn.layer_norm(hin, (hin.shape[-1],), leaves["norm.weight"], leaves["norm.bias"], 1e-5)

    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        out = objective(*[emb(i, m, sd_) for (i, m), sd_ in zip(batches, seeds)])
        out.backward()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    g = {k: v.grad for k, v in leaves.items()}
    g["roberta.embeddings.word_embeddings.weight"][pad] = 0
    g["roberta.embeddings.position_embeddings.weight"][pad] = 0
    return float(out.detach()), g
