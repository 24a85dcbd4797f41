"""fp64 mirror of the encoder backward's orchestration (backward_impl in csrc/encoder.cu), one stage at a time, with a
written per-element bound for every output.

Each stage starts from what the kernel itself saw: the 16-bit activations its training forward saved (widened exactly),
the key bias, the weights rounded to operand_fmt as the handle holds them, and the fp32 upstream gradient the backward
captured at the stage's entry (ance_encoder_debug_grads).  So the check does not loosen with depth: layer l is held to
the same kind of bound at 12 layers as at 2.  Stages:
  head_bwd_ref        d_out, head_in (fp32), x_final  ->  head_w / head_b / head_ln_g / head_ln_b,  d x_final
  layer_bwd_ref       dy = d X_out (d x_final in the pruned last layer)  ->  the 16 ance_layer_grads,  d X_in
  embedding_stage_ref d X_0 (slot 0), ids  ->  word / position / type rows, emb_ln_g / emb_ln_b

Rounding steps of the backward, handled two ways:
* deterministic conversions are emulated exactly: the bf16 transposes of 16-bit activations (transpose_bf16<S>, an fp16
  value rounded to nearest bf16; the identity in bf16), the bf16 W^T copies of the operand_fmt weights, and the fp32
  embedding sum (word[id] + pos[p]) + type[0];
* data-dependent roundings (to_bf16 of dT / dA and of dQKV, the bf16 store of dCTX) are emulated on the mirror's own
  value, and the bound says where the kernel's rounding can differ.  Round-to-nearest is monotone, so every fp32 value
  within e of x rounds into [bf16(x - e), bf16(x + e)]: the kernel's operand differs from the mirror's bf16(x) by at most
  hi - lo, which is zero unless a rounding midpoint lies within e of x (one bf16 spacing when one does).
  Propagating |bf16(x) - x| <= 2^-8 |x| instead (bf16 keeps 8 significant bits) does not work as a bound here: through
  the absolute values of a K-term GEMM it grows ~2^-8 sqrt(K) relative per GEMM, and by the LN1 backward of one layer it
  exceeds the gradients themselves, so it could not reject any orchestration bug downstream.

Error model (u = 2^-24; a quantity with exact value x and computed value x~ carries a bound e >= |x~ - x| elementwise;
|x|+e bounds |x~|; all propagation runs through absolute values, so no cancellation is assumed anywhere):
* bf16 rounding of a computed operand:      x' = bf16(x),  e' = bf16(x + e) - bf16(x - e)
* GEMM C = A B over K terms (A computed, B an exact bf16 operand), fp32 accumulation (tests/encoder_grad_refs.gemm_tol):
      e_C = e_A |B| + gamma_(K+2) (|A| + e_A) |B|
* LayerNorm backward dx = J(x) dy (J linear in dy): encoder_grad_refs.ln_bwd_tol evaluated at |dy| + e_dy, plus the
  propagated input error  rstd (|gamma| e + mean(|gamma| e) + |xhat| mean(|gamma| e |xhat|))  for dx, sum e |xhat| for
  dgamma, sum e for dbeta and the column sum of the dx term for the bias gradient.
* GELU backward dU = dF * g'(u) (one fp32 product):  e_dF (|g'| + t) + |dF| t + u (|dF| + e_dF)(|g'| + t),
  t = encoder_grad_refs.gelu_bwd_tol(u).
* attention backward: linear in dO, so the dO error is propagated through the magnitudes of that map
      |dV| <- P^T e,  |dP| <- e |V|^T,  |dS| <- P o (|dP| + rowsum(P o |dP|)),  |dQ| <- |dS| |K| / 8,  |dK| <- |dS|^T |Q| / 8
  plus encoder_grad_refs.attention_bwd_tol evaluated at |dO| + e.
* column sums (colsum: `per` rows in order in each of `chunks` chunks, then the chunks in order): gamma_(per+chunks+1)
  sum |x| + sum e.
* residual adds (add_rows): e_a + e_b + u (|a + b| + e_a + e_b).
* embedding scatter: encoder_grad_refs.embedding_grads_tol at |dE| + e, plus the scatter of e.
Each stage's bound is its own function of its inputs, so a rewrite of one kernel (split-K wgrad, a tensor-core attention
backward) changes one term.

Perturbed mirrors model orchestration bugs (layer_bwd_ref / head_bwd_ref `perturb`); the tests say which of them the
bound rejects on their data:
  "ln1_residual_rows"  last layer: the LN1 residual gradient added to rows 0 .. B-1 instead of the CLS rows b L
  "wo_ctx_pitch"       last layer: the Wo wgrad reads CTX at pitch H (rows 0 .. B-1) instead of L H
  "gelu_at_ff"         the GELU derivative taken at the GELU output FF instead of the pre-activation U
  "qk_bias_swap"       the q and k bias gradients swapped
  "no_ffn_residual"    dX1 without the FFN residual (add_rows(dX1 += dT) missing)
  "head_x_pitch"       head: the wgrad reads X at pitch L H (rows b L of the buffer that starts at x_final)
and, on a packed plan (ance_encoder_forward_train_packed; `plan` below), the packed path's own index work:
  "cls_residual_dense_rows"  last layer: the LN1 residual lands at rows b L < M (what add_rows does without seq_row0)
  "wo_ctx_packed_rows"       last layer: the Wo wgrad reads rows 0 .. B-1 of the packed CTX instead of cls_ctx
  "attention_whole_tile"     L <= 128: each tile's real rows attend as one sequence (a lost per-sequence bound)
  "position_from_row"        embeddings: position ids counted from the row's offset in its tile (embedding_stage_ref)
  "hidden_mask_by_row"       dropout: hidden masks keyed by the packed row instead of its token
                             (encoder_dropout_refs.packed_hidden_mask)
  "attn_mask_from_tile"      dropout: attention mask counters (query, key) start at the tile's first row instead of the
                             sequence's (encoder_dropout_refs.packed_attn_masks)

A packed plan = (seq_row0 [B], seq_len [B], row_tok [M], M): the layers' rows are the M packed rows as the forward saved
them (row r is the dense token row_tok[r], -1 for a row of no sequence).  Row-wise stages run on those rows unchanged, and
column sums and weight gradients over all M of them, as the kernels do.  The attention stage gathers each sequence's
rows to dense positions b L + i (the keys past seq_len[b] masked), runs the dense stage and scatters the result back:
rows of no sequence, and rows past a sequence's length, get exactly 0.  In the pruned last layer the B compact rows are
the CLS rows seq_row0[b]: the Wo wgrad reads cls_ctx and the LN1 residual goes into d X_in at seq_row0[b].
"""
from __future__ import annotations

import torch

from tests import encoder_grad_refs as G

F64 = torch.float64
U32 = 2.0 ** -24
TINY = 1e-30

LAYER_GRADS = ("q_w", "q_b", "k_w", "k_b", "v_w", "v_b", "ao_w", "ao_b", "ln1_g", "ln1_b",
               "ff1_w", "ff1_b", "ff2_w", "ff2_b", "ln2_g", "ln2_b")
HEAD_GRADS = ("head_w", "head_b", "head_ln_g", "head_ln_b")


def to_bf16(x):
    """bf16 round-to-nearest of a 16-bit or fp32 value, as transpose_bf16_kernel / f32_to_bf16_kernel do it."""
    return x.to(torch.float32).to(torch.bfloat16).to(F64)


def _rnd(x, e, exact):
    """A computed operand rounded to bf16 (data-dependent) -> (the mirror's operand, its bound); see the module doc."""
    if exact:
        return x, e
    return to_bf16(x), to_bf16(x + e) - to_bf16(x - e)


def _mm(a, ea, b, exact=False):
    """(a @ b, bound) for a computed a (bound ea) and an exact operand b, fp32 accumulation over K terms."""
    ab = b.abs()
    K = a.shape[1]
    return a @ b, ea @ ab + G._g(K + 2) * ((a.abs() + ea) @ ab) + TINY


def _colsum(x, ex):
    rows = x.shape[0]
    chunks = min(rows, 128)
    per = -(-rows // chunks)
    chunks = -(-rows // per)
    return x.sum(0), G._g(per + chunks + 1) * (x.abs() + ex).sum(0) + ex.sum(0) + TINY


def _add(a, ea, b, eb):
    s = a + b
    return s, ea + eb + U32 * (s.abs() + ea + eb)


def ln_stage(x, gamma, eps, dy, edy):
    """LayerNorm backward with an upstream gradient that carries the bound edy -> ((dx, dgamma, dbeta, dsum), bounds)."""
    x, gamma = x.to(F64), gamma.to(F64)
    vals = G.ln_bwd_ref(x, gamma, eps, dy)
    tdx, tg, tb, ts = G.ln_bwd_tol(x, gamma, eps, dy.abs() + edy)
    mean = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + eps)
    xh = ((x - mean) * rstd).abs()
    ge = edy * gamma.abs()
    pdx = rstd * (ge + ge.mean(-1, keepdim=True) + xh * (ge * xh).mean(-1, keepdim=True))
    return vals, (tdx + pdx, tg + (edy * xh).sum(0), tb + edy.sum(0), ts + pdx.sum(0))


def _attention_abs(qkv, kbias, a, B, L, heads):
    """|dQKV| <- the magnitudes of the attention backward's linear map in dO, applied to a >= 0."""
    q, k, v = G._split(qkv.to(F64).abs(), B, L, heads)
    p = G.attention_probs(qkv, kbias, B, L, heads)
    do = a.reshape(B, L, heads, 64).transpose(1, 2)
    adp = do @ v.transpose(-1, -2)
    ads = p * (adp + (p * adp).sum(-1, keepdim=True))
    return torch.cat([G._merge(ads @ k / 8.0, B, L, heads), G._merge(ads.transpose(-1, -2) @ q / 8.0, B, L, heads),
                      G._merge(p.transpose(-1, -2) @ do, B, L, heads)], dim=1)


def attention_stage(qkv, kbias, dout, edout, B, L, heads):
    ref = G.attention_bwd_ref(qkv, kbias, dout, B, L, heads)
    tol = G.attention_bwd_tol(qkv, kbias, dout.abs() + edout, B, L, heads) + _attention_abs(qkv, kbias, edout, B, L, heads)
    return ref, tol


def strided_rows(flat, rows, H, pitch):
    """rows x H elements of a flat buffer read at row pitch `pitch` (elements); rows past its end read as zeros."""
    out = torch.zeros(rows, H, dtype=flat.dtype, device=flat.device)
    for r in range(rows):
        o = r * pitch
        n = max(0, min(H, flat.numel() - o))
        out[r, :n] = flat[o:o + n]
    return out


LOG2_MASK = -10000.0 * 1.4426950408889634   # the key bias of a padding key (log2 units)


def plan_rows(plan, L):
    """(packed rows, dense rows b L + i) of the tokens i < seq_len[b] of every sequence of a packed plan."""
    row0, lens = plan[0], plan[1]
    pr = [int(row0[b]) + torch.arange(int(lens[b])) for b in range(len(row0))]
    dr = [b * L + torch.arange(int(lens[b])) for b in range(len(row0))]
    return torch.cat(pr), torch.cat(dr)


def packed_attention(stage, qkv, kbias, dout, edout, B, L, heads, plan, whole_tile=False):
    """stage(qkv, kbias, dout, edout, B, L, heads) -> (dQKV, bound), a dense attention stage, run on the M packed rows of
    a plan: each sequence gathered to rows b L + i (keys past its length masked), the result scattered back; rows of no
    sequence and rows past a sequence's length get exactly 0.  whole_tile (the "attention_whole_tile" perturbation, L <=
    128): each 128-row tile's real rows attend as one sequence."""
    dev, M, H3 = qkv.device, plan[3], qkv.shape[1]
    if whole_tile:
        tok = plan[2].to(dev).long()
        real = (tok >= 0) & ((tok % L) < plan[1].to(dev).long()[tok.clamp(min=0) // L])
        ref, tol = stage(qkv, torch.where(real, kbias.to(F64), LOG2_MASK), dout, edout, M // 128, 128, heads)
        return ref * real[:, None], tol * real[:, None]
    pr, dr = (t.to(dev) for t in plan_rows(plan, L))
    n, H = B * L, dout.shape[1]
    q = torch.zeros(n, H3, dtype=F64, device=dev)
    kb = torch.full((n,), LOG2_MASK, dtype=F64, device=dev)
    do, eo = torch.zeros(n, H, dtype=F64, device=dev), torch.zeros(n, H, dtype=F64, device=dev)
    q[dr], kb[dr], do[dr], eo[dr] = qkv[pr].to(F64), kbias[pr].to(F64), dout[pr], edout[pr]
    ref, tol = stage(q, kb, do, eo, B, L, heads)
    out, eout = torch.zeros(M, H3, dtype=F64, device=dev), torch.zeros(M, H3, dtype=F64, device=dev)
    out[pr], eout[pr] = ref[dr], tol[dr]
    return out, eout


def last_ctx(act, B, L, plan, perturb):
    """The rows the pruned last layer's Wo wgrad reads: the CLS rows of CTX (dense: at pitch L H; packed: cls_ctx, the
    rows seq_row0 that the forward gathered)."""
    ctx = act["ctx"]
    if plan is None:
        return ctx[:B] if perturb == "wo_ctx_pitch" else ctx.reshape(B, L, -1)[:, 0]
    if perturb == "wo_ctx_packed_rows":
        return ctx[:B]
    return act["cls_ctx"] if "cls_ctx" in act else ctx[plan[0].to(ctx.device).long()]


def cls_rows(B, L, M, plan, perturb=None, dev=None):
    """(rows of the M-row stream, which of the B compact rows land there) of the pruned last layer's CLS rows."""
    r = torch.arange(B, device=dev) * L
    if plan is not None and perturb != "cls_residual_dense_rows":
        r = plan[0].to(dev).long()
    keep = r < M
    return r[keep], keep


def layer_bwd_ref(act, kbias, w, dy, B, L, heads, last, eps, exact=False, perturb=None, plan=None):
    """One layer of backward_impl.

    act: the layer's saved activations widened to fp64 — x_in [M, H], qkv [M, 3H], ctx [M, H] (M = B L) and t1, x1, u,
    ff, t2 [Mr, .] (Mr = B in the pruned last layer, whose rows are then the CLS rows, else M); kbias [M] in log2 units;
    w: wqkv [3H, H], wo [H, H], w1 [F, H], w2 [H, F] as operand_fmt values (fp64), ln1_g / ln2_g [H]; dy [Mr, H] the fp32
    upstream gradient.  exact=True skips the deterministic bf16 conversions (the exact-arithmetic chain, for autograd).
    plan = (seq_row0, seq_len, row_tok, M): the layer ran a packed plan (see the module doc); M is then the plan's row
    count and act may carry cls_ctx [B, H], the last layer's gathered CTX rows.
    -> (grads, bounds): dicts over LAYER_GRADS + ("x_in",), x_in the gradient into the layer input [M, H]."""
    cv = (lambda t: t.to(F64)) if exact else to_bf16
    dy = dy.to(F64)
    M = B * L if plan is None else plan[3]
    Mr = B if last else M
    zero = lambda t: torch.zeros_like(t)
    g, t = {}, {}
    # LN2: T2 = FF W2^T + b2 + X1
    (dT, g["ln2_g"], g["ln2_b"], g["ff2_b"]), (eT, t["ln2_g"], t["ln2_b"], t["ff2_b"]) = ln_stage(
        act["t2"], w["ln2_g"], eps, dy, zero(dy))
    A, eA = _rnd(dT, eT, exact)
    g["ff2_w"], t["ff2_w"] = _mm(A.t(), eA.t(), cv(act["ff"]))
    dF, eF = _mm(A, eA, cv(w["w2"]))
    # GELU: dU = dF * gelu'(u)
    gu = act["u"] if perturb != "gelu_at_ff" else act["ff"]
    d = G.gelu_bwd_ref(gu)
    td = G.gelu_bwd_tol(act["u"])
    dU = dF * d
    eU = eF * (d.abs() + td) + dF.abs() * td + U32 * (dF.abs() + eF) * (d.abs() + td)
    g["ff1_b"], t["ff1_b"] = _colsum(dU, eU)
    A, eA = _rnd(dU, eU, exact)
    g["ff1_w"], t["ff1_w"] = _mm(A.t(), eA.t(), cv(act["x1"]))
    dX1, eX1 = _mm(A, eA, cv(w["w1"]))
    if perturb != "no_ffn_residual":
        dX1, eX1 = _add(dX1, eX1, dT, eT)
    # LN1: T1 = CTX Wo^T + bo + X_in
    (dT1, g["ln1_g"], g["ln1_b"], g["ao_b"]), (eT1, t["ln1_g"], t["ln1_b"], t["ao_b"]) = ln_stage(
        act["t1"], w["ln1_g"], eps, dX1, eX1)
    A, eA = _rnd(dT1, eT1, exact)
    ctx = last_ctx(act, B, L, plan, perturb) if last else act["ctx"]
    g["ao_w"], t["ao_w"] = _mm(A.t(), eA.t(), cv(ctx))
    dC, eC = _rnd(*_mm(A, eA, cv(w["wo"])), exact)   # dCTX is stored bf16
    H = dC.shape[1]
    if last:   # cls_only: the gradient of token 0 of every sequence, none elsewhere
        dO, eO = torch.zeros(M, H, dtype=F64, device=dC.device), torch.zeros(M, H, dtype=F64, device=dC.device)
        if plan is None:
            dO[::L], eO[::L] = dC, eC
        else:
            r0 = plan[0].to(dC.device).long()
            dO[r0], eO[r0] = dC, eC
    else:
        dO, eO = dC, eC
    # attention -> dQKV [M, 3H]
    if plan is None:
        dA, eA3 = attention_stage(act["qkv"], kbias, dO, eO, B, L, heads)
    else:
        dA, eA3 = packed_attention(attention_stage, act["qkv"], kbias, dO, eO, B, L, heads, plan,
                                   whole_tile=perturb == "attention_whole_tile")
    bq, tq = _colsum(dA, eA3)
    g["q_b"], g["k_b"], g["v_b"] = bq[:H], bq[H:2 * H], bq[2 * H:]
    t["q_b"], t["k_b"], t["v_b"] = tq[:H], tq[H:2 * H], tq[2 * H:]
    if perturb == "qk_bias_swap":
        g["q_b"], g["k_b"] = g["k_b"], g["q_b"]
    A, eA = _rnd(dA, eA3, exact)
    xt = cv(act["x_in"])
    for i, n in enumerate(("q_w", "k_w", "v_w")):
        s = slice(i * H, (i + 1) * H)
        g[n], t[n] = _mm(A[:, s].t(), eA[:, s].t(), xt)
    dX, eX = _mm(A, eA, cv(w["wqkv"]))
    dX, eX = dX.clone(), eX.clone()
    if last and plan is not None:
        rows, keep = cls_rows(B, L, M, plan, perturb, dX.device)
        dX[rows], eX[rows] = _add(dX[rows], eX[rows], dT1[keep], eT1[keep])
    else:
        rows = slice(0, B) if (last and perturb == "ln1_residual_rows") else slice(None, None, L) if last else slice(None)
        dX[rows], eX[rows] = _add(dX[rows], eX[rows], dT1, eT1)
    g["x_in"], t["x_in"] = dX, eX
    return g, t


def head_bwd_ref(d_out, head_in, x_final, head_w, head_g, exact=False, perturb=None, x_flat=None, L=None):
    """The head out = LN(x_final Wh^T + bh) (head_in = its fp32 LayerNorm input, eps 1e-5): d_out [B, H] fp32, x_final
    [B, H] 16-bit, head_w [H, H] as operand_fmt values.  -> (grads, bounds) over HEAD_GRADS + ("x_final",).
    perturb "head_x_pitch" reads the wgrad's X rows at pitch L H from x_flat (the 16-bit buffer that starts at x_final)."""
    cv = (lambda t: t.to(F64)) if exact else to_bf16
    d_out = d_out.to(F64)
    g, t = {}, {}
    (dT, g["head_ln_g"], g["head_ln_b"], g["head_b"]), (eT, t["head_ln_g"], t["head_ln_b"], t["head_b"]) = ln_stage(
        head_in, head_g, 1e-5, d_out, torch.zeros_like(d_out))
    A, eA = _rnd(dT, eT, exact)
    B, H = x_final.shape
    x = x_final if perturb != "head_x_pitch" else strided_rows(x_flat, B, H, L * H)
    g["head_w"], t["head_w"] = _mm(A.t(), eA.t(), cv(x))
    g["x_final"], t["x_final"] = _mm(A, eA, cv(head_w))
    return g, t


def embedding_sum(ids, word, pos, typ, pad_id, roberta, max_pos, pos_shift=0):
    """E = (word[id] + pos[p]) + type[0] in the tables' precision (fp32 tables: exactly embed_sum_kernel's values)."""
    p = (G.position_ids(ids.long().cpu(), pad_id, roberta) + pos_shift).clamp(0, max_pos - 1).to(word.device)
    return (word[ids.long()] + pos[p]) + typ[0]


def packed_to_dense(x, row_tok, n):
    """Rows [M, .] of a packed plan scattered to their dense tokens (row r to row_tok[r]) of an n-row zero matrix."""
    tok = row_tok.to(x.device).long()
    out = torch.zeros(n, x.shape[1], dtype=x.dtype, device=x.device)
    out[tok[tok >= 0]] = x[tok >= 0]
    return out


def position_from_row_shift(plan, lens, B, L):
    """pos_shift [B, L] of the "position_from_row" perturbation: token i < lens[b] of sequence b at its row's offset in
    its tile, (seq_row0[b] + i) mod 128, instead of i."""
    i = torch.arange(L)[None, :]
    shift = (plan[0].long().cpu()[:, None] + i) % 128 - i
    return torch.where(i < torch.as_tensor(lens).long()[:, None], shift, 0)


def embedding_stage_ref(ids, dx0, word, pos, typ, emb_g, eps, pad_id, roberta, pos_shift=0):
    """d X_0 [B L, H] (slot 0) through the embedding LayerNorm into the tables.  -> (grads, bounds) over word_emb,
    pos_emb, type_emb (row 0 = the LayerNorm's column sum of dE; the other rows get nothing), emb_ln_g, emb_ln_b.
    dx0 holds dense rows: the caller scatters a packed plan's slot 0 to its dense tokens first (packed_to_dense).
    pos_shift [B, L] (a perturbation) moves the position ids."""
    vocab, max_pos, H = word.shape[0], pos.shape[0], word.shape[1]
    E = embedding_sum(ids, word, pos, typ, pad_id, roberta, max_pos, pos_shift).reshape(-1, H)
    dx0 = dx0.to(F64)
    (dE, dg, db, ds), (eE, tg, tb, ts) = ln_stage(E, emb_g, eps, dx0, torch.zeros_like(dx0))
    idc = ids.long().cpu()
    dw, dp = G.embedding_grads_ref(idc, dE.cpu(), vocab, max_pos, pad_id, roberta, pos_shift)
    tw, tp = G.embedding_grads_tol(idc, (dE.abs() + eE).cpu(), vocab, max_pos, pad_id, roberta)
    ew, ep = G.embedding_grads_ref(idc, eE.cpu(), vocab, max_pos, pad_id, roberta)   # the scatter of the dE bound
    dt = torch.zeros(typ.shape[0], H, dtype=F64, device=dE.device)
    tt = torch.full_like(dt, TINY)
    dt[0], tt[0] = ds, ts
    dev = dE.device
    g = {"word_emb": dw.to(dev), "pos_emb": dp.to(dev), "type_emb": dt, "emb_ln_g": dg, "emb_ln_b": db}
    t = {"word_emb": (tw + ew).to(dev), "pos_emb": (tp + ep).to(dev), "type_emb": tt, "emb_ln_g": tg, "emb_ln_b": tb}
    return g, t


def construct_for_discrimination(sd, n_layer, prefix):
    """Weights on which every orchestration perturbation above shows.  Query weights and bias
    / 16 and key weights and bias x 16 leave every score Q K^T unchanged (powers of two: exactly), but make dQ 16x and dK
    1/16x as large, so the q bias gradient stands far above the k bias gradient's bound (a q / k swap shows; on random
    weights the q bias gradient is a sum over heavily cancelling dS rows and sits inside that bound).  The out-projection
    / 64 shrinks the attention path's contribution to d X_in, and its bound, next to the LN1 residual (a residual added to
    the wrong rows shows).  Modifies sd in place."""
    for l in range(n_layer):
        p = f"{prefix}encoder.layer.{l}."
        for n in ("query.weight", "query.bias"):
            sd[p + "attention.self." + n] /= 16.0
        for n in ("key.weight", "key.bias"):
            sd[p + "attention.self." + n] *= 16.0
        sd[p + "attention.output.dense.weight"] /= 64.0
    return sd
