"""Packed training backward layer by layer on the GPU: every gradient element of every layer, the head and the embedding
stage of ance_encoder_forward_train_packed + ance_encoder_backward against the plan-aware fp64 mirror of
tests/encoder_layer_refs.py / encoder_dropout_refs.py, fed the kernel's own saved activations (located by
ance_dbg_train_layout_packed) and its own captured upstream gradients, at varlen_align 16 and 1, with and without
dropout.  Also: the plan the workspace holds equals the host planner's, the gathered CLS rows are the CTX rows they were
gathered from, rows of no sequence carry exactly zero gradient, and at align 16 every captured row of a real token is the
dense backward's row of the same token, bit for bit."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from ance_b200 import _lib
from ance_b200.models import _backbone
from tests import encoder_dropout_refs as D
from tests import encoder_grad_long_refs as R
from tests import encoder_layer_refs as LR
from tests.test_gpu_encoder_backward import FMT_CODE
from tests.test_gpu_encoder_backward_layers import DT16, VOCAB, _d_out, _Enc, _roberta, _w16

pytestmark = pytest.mark.gpu

F64 = torch.float64
FMTS = ["fp16", "bf16"]
P = 0.1
CAPTURE_ROWS = 4096   # ance_encoder_debug_grads keeps the slots of backwards of up to this many rows

# Rejected wherever they change the mirror (asserted per call: some stage of the call puts the kernel outside the bound
# around the perturbed mirror).  "attention_whole_tile" and "attn_mask_from_tile" change only the attention backward's
# inner arithmetic; through a layer they stay inside the attention stage's propagated bound (the upstream gradient's
# bf16 rounding, carried through the absolute values of the attention map), so each call also runs the per-sequence
# attention kernel on its own plan and layer-0 QKV with an exact upstream gradient (_attention_on_the_plan), where the
# bound has no upstream term and both are rejected, at align 1 as at align 16.
ASSERTED = ("gelu_at_ff", "no_ffn_residual", "wo_ctx_packed_rows", "position_from_row", "hidden_mask_by_row",
            "attention_whole_tile", "attn_mask_from_tile", "no_mask_bwd", "no_scale_bwd", "residual_masked",
            "bias_unmasked", "embedding mask not applied")
# "cls_residual_dense_rows", the packed form of the dense suite's "ln1_residual_rows", stays inside the last layer's
# d X_in bound (0.17 .. 0.85 on these weights).  At align 16 it is rejected by the bit equality of every captured row
# with the dense backward's (_dense_rows_equal): the residual at rows b L instead of seq_row0[b] leaves the CLS row of a
# sequence with seq_row0[b] != b L without it, so that row differs from the dense row of token b L.  Printed at align 1.
EQUALITY_HELD = ("cls_residual_dense_rows",)
# Printed only: "qk_bias_swap" (inside the k bias gradient's bound on random weights, as in
# tests/test_gpu_encoder_backward_layers.py) and the dropout mirror's "d_unmasked" / "mask_transposed" (asserted on the
# kernel itself in tests/test_gpu_encoder_dropout.py).


@pytest.fixture(scope="module")
def gpu_lib():
    assert torch.cuda.is_available()
    return _lib.load()


class _Report:
    """Worst error / bound per stage.  Per call, the largest err / bound of each perturbation over the stages where it
    changes the mirror (a perturbation that is a no-op on a plan is skipped); over calls, the smallest of those."""

    def __init__(self, asserted=ASSERTED):
        self.worst, self.pert, self.asserted, self.call, self.held = {}, {}, asserted, {}, {}

    def check(self, stage, name, out, g, t, perturbed=()):
        for k in g:
            err = float(((out[k].double() - g[k]).abs() / t[k]).max())
            assert err <= 1.0, (name, stage, k, err)
            self.worst[stage] = max(self.worst.get(stage, 0.0), err)
        for pn, gp in dict(perturbed).items():
            if all(torch.equal(gp[k], g[k]) for k in g):
                continue
            rep = max(float(((out[k].double() - gp[k]).abs() / t[k]).max()) for k in g)
            self.call[pn] = max(self.call.get(pn, 0.0), rep)

    def end_call(self, name, dense_equal=False):
        """dense_equal: the call's captured rows equal the dense backward's bit for bit, which rejects EQUALITY_HELD."""
        for pn, rep in self.call.items():
            ok = rep > 1.0 or pn not in self.asserted or (dense_equal and pn in EQUALITY_HELD)
            assert ok, (name, pn, rep)
            self.pert[pn] = min(self.pert.get(pn, math.inf), rep)
            if dense_equal and pn in EQUALITY_HELD:
                self.held[pn] = self.held.get(pn, 0) + 1
        self.call = {}

    def show(self, name):
        print(f"{name}: worst err / bound {({k: round(v, 3) for k, v in self.worst.items()})}; "
              f"smallest perturbed err / bound {({k: round(v, 2) for k, v in self.pert.items()})}; "
              f"calls rejecting by dense equality {self.held}")


def _layout(e, lens, B, L):
    """ance_dbg_train_layout_packed at the handle's current varlen_align -> (train fields, packed fields, n_tiles)."""
    out = (C.c_size_t * (len(_lib.TRAIN_LAYOUT_FIELDS) + len(_lib.PACKED_LAYOUT_FIELDS)))()
    n = C.c_int()
    lh = lens.to(torch.int32).contiguous()
    _lib.check(e.enc.lib.ance_dbg_train_layout_packed(e.enc.h, lh.data_ptr(), B, L, out, C.byref(n)))
    k = len(_lib.TRAIN_LAYOUT_FIELDS)
    return dict(zip(_lib.TRAIN_LAYOUT_FIELDS, out[:k])), dict(zip(_lib.PACKED_LAYOUT_FIELDS, out[k:])), n.value


def _pack_rows(lib, lens, L, max_tokens, align):
    B = len(lens)
    ln = lens.to(torch.int32).numpy()
    row0 = np.zeros(B, np.int32)
    tok = np.full(max_tokens, -7, np.int32)
    n_placed, n_tiles = C.c_int(), C.c_int()
    assert lib.ance_dbg_pack_rows(ln.ctypes.data, B, L, max_tokens, align, row0.ctypes.data, tok.ctypes.data,
                                  C.byref(n_placed), C.byref(n_tiles)) == 0
    assert n_placed.value == B
    return torch.from_numpy(row0).long(), torch.from_numpy(tok[:n_tiles.value * 128].copy()).long(), n_tiles.value


def _backward(e, ws, d_out):
    embs, layers, hd = e.groups
    mk = lambda ts: [torch.full(t.shape, float("nan"), device="cuda") for t in ts]
    grads = (mk(embs), [mk(l) for l in layers], mk(hd))
    e.enc.backward(d_out, ws, grads)
    slots = []
    for s in range(e.n_layer + 1):
        buf = torch.empty(CAPTURE_ROWS, e.H, device="cuda")
        _lib.check(e.enc.lib.ance_encoder_debug_grads(e.enc.h, s, buf.data_ptr(), _lib.current_stream()))
        slots.append(buf)
    torch.cuda.synchronize()
    return grads, slots


def _forward(e, ids, lens, align, drop=None):
    """The packed training forward, and its workspace layout queried right after it (forward_train_packed has just set
    the handle's varlen_align to `align`).  -> (workspace, layout)."""
    lh = lens.to(torch.int32)
    _, ws = e.enc.forward_train_packed(ids.to(torch.int32).cuda(), lh.cuda(), lh, drop, align=align)
    return ws, _layout(e, lens, *ids.shape)


def _long_stage(fmt):
    short = LR.attention_stage

    def stage(qkv, kbias, dout, edout, B, L, heads):
        if L <= 128:
            return short(qkv, kbias, dout, edout, B, L, heads)
        return R.attention_stage(qkv, kbias, dout, edout, B, L, heads, fmt)
    return stage


def _check_ws(e, ids, lens, fwd, d_out, rep, name, align, drop=None, dense_equal=True):
    """The backward of the packed forward fwd = _forward(...) (its workspace and layout), every stage against the mirror
    (see the module doc).  The handle's varlen_align is whatever the last forward left: the backward reads the plan of
    its own workspace."""
    B, L = ids.shape
    H, fmt, NL, heads = e.H, e.fmt, e.n_layer, e.heads
    ws, (lo, pk, n_tiles) = fwd
    M = n_tiles * 128
    assert M <= CAPTURE_ROWS and pk["total"] == ws.numel()
    grads, slots = _backward(e, ws, d_out)
    # the plan the workspace holds: the host planner's
    i32 = lambda off, n: ws[off:off + 4 * n].view(torch.int32).cpu().long()
    row0, seq_len, row_tok = i32(pk["seq_row0"], B), i32(pk["seq_len"], B), i32(pk["row_tok"], M)
    want0, want_tok, want_tiles = _pack_rows(e.enc.lib, lens, L, e.enc.max_tokens, align)
    assert want_tiles == n_tiles and torch.equal(row0, want0) and torch.equal(row_tok, want_tok), name
    assert torch.equal(seq_len, lens.long()), name
    kb = ws[lo["kbias"]:lo["kbias"] + M * 4].view(torch.float32)
    assert torch.count_nonzero(kb) == 0, name
    kb = kb.to(F64)
    plan = (row0, seq_len, row_tok, M)
    real = (row_tok >= 0) & ((row_tok % L) < lens.long()[row_tok.clamp(min=0) // L])
    for s in range(NL):
        assert torch.count_nonzero(slots[s][:M][~real.cuda()]) == 0, (name, "rows of no token", s)
    a16 = lambda off, rows, cols: ws[off:off + rows * cols * 2].view(DT16[fmt]).view(rows, cols)
    _attention_on_the_plan(e, a16(lo["layers"] + lo["qkv"], M, 3 * H), kb, plan, B, L, drop, rep, name)
    # the gathered CLS rows of the last layer: its CTX and X_in rows at seq_row0, bit for bit
    base = lo["layers"] + (NL - 1) * lo["per_layer"]
    r0 = row0.cuda()
    assert torch.equal(a16(pk["cls_ctx"], B, H).view(torch.int16), a16(base + lo["ctx"], M, H)[r0].view(torch.int16))
    assert torch.equal(a16(pk["cls_x"], B, H).view(torch.int16), a16(base + lo["x_in"], M, H)[r0].view(torch.int16))
    embs, layers, hd = e.groups
    gembs, glayers, ghd = grads
    seed = None if drop is None else drop[2]
    p_attn = 0.0 if drop is None else drop[1]
    s = D.scale(P)
    x_final = a16(lo["x_final"], B, H).to(F64)
    if hd:
        head_in = ws[lo["head_in"]:lo["head_in"] + B * H * 4].view(torch.float32).view(B, H).to(F64)
        g, t = LR.head_bwd_ref(d_out, head_in, x_final, _w16(hd[0], fmt), hd[2].detach())
        rep.check("head", name + " head", dict(zip(LR.HEAD_GRADS, ghd), x_final=slots[NL][:B]), g, t)
    else:
        assert torch.equal(slots[NL][:B], d_out)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(LR, "attention_stage", _long_stage(fmt))
        for l in reversed(range(NL)):
            last = l == NL - 1
            Mr = B if last else M
            base = lo["layers"] + l * lo["per_layer"]
            F = layers[l][10].shape[0]
            act = {"x_in": a16(base + lo["x_in"], M, H), "qkv": a16(base + lo["qkv"], M, 3 * H),
                   "ctx": a16(base + lo["ctx"], M, H), "t1": a16(base + lo["t1"], Mr, H),
                   "x1": a16(base + lo["x1"], Mr, H), "u": a16(base + lo["u"], Mr, F), "ff": a16(base + lo["ff"], Mr, F),
                   "t2": a16(base + lo["t2"], Mr, H)}
            act = {k: v.to(F64) for k, v in act.items()}
            if last:
                act["cls_ctx"] = a16(pk["cls_ctx"], B, H).to(F64)
            p = layers[l]
            w = {"wqkv": _w16(torch.cat([p[0], p[2], p[4]]), fmt), "wo": _w16(p[6], fmt), "w1": _w16(p[10], fmt),
                 "w2": _w16(p[12], fmt), "ln1_g": p[8].detach(), "ln2_g": p[14].detach()}
            dy = slots[l + 1][:Mr]
            out = dict(zip(LR.LAYER_GRADS, glayers[l]), x_in=slots[l][:M])
            names = ["cls_residual_dense_rows", "wo_ctx_packed_rows"] if last and B > 1 else []
            if seed is None:
                names += ["gelu_at_ff", "no_ffn_residual", "qk_bias_swap"]
                if L <= 128 and (last or l == 0):
                    names.append("attention_whole_tile")
                g, t = LR.layer_bwd_ref(act, kb, w, dy, B, L, heads, last, e.eps, plan=plan)
                pert = {n: LR.layer_bwd_ref(act, kb, w, dy, B, L, heads, last, e.eps, perturb=n, plan=plan)[0]
                        for n in names}
            else:
                def masks(pm=None):
                    if last:
                        hm = [D.hidden_mask(seed, site, l, np.arange(B) * L, H, P) for site in (2, 3)]
                    else:
                        hm = [D.packed_hidden_mask(seed, site, l, row_tok.numpy(), H, P, pm) for site in (2, 3)]
                    am = D.packed_attn_masks(seed, l, B, heads, L, p_attn, row0.numpy(), pm) if p_attn > 0 else \
                        np.ones((B, heads, L, L))
                    return [torch.tensor(x, device="cuda") for x in hm] + [torch.tensor(am, device="cuda")]
                sc = s if p_attn > 0 else 1.0
                args = lambda pm=None: (act, kb, w, dy, B, L, heads, last, e.eps, fmt, *masks(pm))
                # hidden sites at p_hidden: the mirror takes one scale, so p_attn is either P or 0 (then its mask is
                # all ones and its scale 1, the unmasked attention exactly)
                g, t = _masked(args(), s, sc, plan)
                pert = {n: _masked(args(), s, sc, plan, n)[0] for n in names + list(D.PERTURBATIONS)}
                if l == 0:
                    pert["hidden_mask_by_row"] = _masked(args("hidden_mask_by_row"), s, sc, plan)[0]
                    if p_attn > 0:
                        pert["attn_mask_from_tile"] = _masked(args("attn_mask_from_tile"), s, sc, plan)[0]
            rep.check("layer", f"{name} layer {l}", out, g, t, pert)
    # embeddings: slot 0 scattered to the dense tokens
    dx0 = LR.packed_to_dense(slots[0][:M], row_tok, B * L)
    eargs = [x.detach() for x in embs[:4]]
    shift = LR.position_from_row_shift(plan, lens, B, L)
    pert = {}
    if seed is not None:
        m0 = torch.tensor(D.hidden_mask(seed, 0, 0, np.arange(B * L), H, P), dtype=torch.float32, device="cuda")
        mr = LR.packed_to_dense(torch.tensor(D.hidden_mask(seed, 0, 0, np.arange(M), H, P), dtype=torch.float32,
                                             device="cuda"), row_tok, B * L)
        sf = torch.tensor(s, dtype=torch.float32)
        pert["embedding mask not applied"] = LR.embedding_stage_ref(ids.cuda(), dx0, *eargs, e.eps, e.pad, e.roberta)[0]
        pert["hidden_mask_by_row"] = LR.embedding_stage_ref(ids.cuda(), (dx0 * sf) * mr, *eargs, e.eps, e.pad,
                                                            e.roberta)[0]
        dx0 = (dx0 * sf) * m0
    g, t = LR.embedding_stage_ref(ids.cuda(), dx0, *eargs, e.eps, e.pad, e.roberta)
    pert["position_from_row"] = LR.embedding_stage_ref(ids.cuda(), dx0, *eargs, e.eps, e.pad, e.roberta,
                                                       pos_shift=shift)[0]
    rep.check("embeddings", name + " embeddings", dict(zip(("word_emb", "pos_emb", "type_emb", "emb_ln_g", "emb_ln_b"),
                                                           gembs)), g, t, pert)
    equal = align == 16 and dense_equal
    if equal:
        assert B * L <= CAPTURE_ROWS, (name, "the dense backward's slots are not captured")
        _dense_rows_equal(e, ids, lens, d_out, drop, slots, row_tok, real, M, name)
    rep.end_call(name, equal)
    return grads


def _attention_on_the_plan(e, qkv16, kb, plan, B, L, drop, rep, name):
    """The per-sequence attention backward (ance_dbg_attention_backward_packed: the launch backward_impl makes) on the
    call's own plan and its layer-0 QKV, with an exact bf16 upstream gradient: every token's query row (cls_only 0) and
    the CLS rows alone (cls_only 1).  Held to the kernel's bound around the dense fp64 reference of each sequence
    (encoder_grad_refs / encoder_grad_long_refs; with attention dropout encoder_dropout_refs' masked reference), rows of
    no token exactly 0; "attention_whole_tile" (L <= 128) and "attn_mask_from_tile" (attention dropout) are rejected
    here."""
    from tests import encoder_grad_refs as G
    fmt, heads, H = e.fmt, e.heads, e.H
    row0, lens, row_tok, M = plan
    p_attn, seed = (0.0, 0) if drop is None else (drop[1], drop[2])
    layer = 0
    s = D.scale(p_attn) if p_attn > 0 else 1.0
    real = (row_tok >= 0) & ((row_tok % L) < lens[row_tok.clamp(min=0) // L])
    g = torch.Generator().manual_seed(M + L)

    def stage_for(am):
        def stage(q, kbias, do, edo, B_, L_, h):
            tol = G.attention_bwd_tol(q, kbias, do, B_, L_, h) if L_ <= 128 else \
                R.attention_bwd_long_tol(q, kbias, do, B_, L_, h, fmt)
            if am is None:
                return G.attention_bwd_ref(q, kbias, do, B_, L_, h), tol
            return D.masked_attention_bwd_ref(q, kbias, do, B_, L_, h, am, s), tol * s * (1 + 4 * 2.0 ** -24)
        return stage
    am = None if p_attn == 0 else torch.tensor(D.attn_masks(seed, layer, B, heads, L, p_attn), device="cuda")
    q64 = qkv16.to(F64)
    for cls_only in (0, 1):
        if cls_only:
            d = torch.randn(B, H, generator=g, dtype=F64).to(torch.bfloat16)
            dfull = torch.zeros(M, H, dtype=torch.bfloat16)
            dfull[row0] = d
        else:
            dfull = (torch.randn(M, H, generator=g, dtype=F64) * real[:, None]).to(torch.bfloat16)
            d = dfull
        dd, do64 = d.cuda(), dfull.to(F64).cuda()
        out = torch.full((M, 3 * H), float("nan"), device="cuda")
        r0, ln, kb32 = row0.to(torch.int32).cuda(), lens.to(torch.int32).cuda(), kb.float().contiguous()
        _lib.check(e.enc.lib.ance_dbg_attention_backward_packed(
            FMT_CODE[fmt], qkv16.data_ptr(), kb32.data_ptr(), dd.data_ptr(), cls_only, B, L, heads, r0.data_ptr(),
            ln.data_ptr(), M, p_attn, seed, layer, out.data_ptr(), _lib.current_stream()))
        torch.cuda.synchronize()
        out = out.double()
        rc = real.cuda()
        assert torch.count_nonzero(out[~rc]) == 0, (name, "attention rows of no token", cls_only)
        z = torch.zeros_like(do64)
        ref, tol = LR.packed_attention(stage_for(am), q64, kb.double(), do64, z, B, L, heads, plan)
        err = float(((out[rc] - ref[rc]).abs() / tol[rc]).max())
        assert err <= 1.0, (name, "attention on the plan", cls_only, err)
        rep.worst["attention on the plan"] = max(rep.worst.get("attention on the plan", 0.0), err)
        perts = {}
        if am is None and L <= 128:
            perts["attention_whole_tile"] = LR.packed_attention(stage_for(None), q64, kb.double(), do64, z, B, L,
                                                                heads, plan, whole_tile=True)[0]
        if am is not None:
            amt = torch.tensor(D.packed_attn_masks(seed, layer, B, heads, L, p_attn, row0.numpy(), "attn_mask_from_tile"),
                               device="cuda")
            perts["attn_mask_from_tile"] = LR.packed_attention(stage_for(amt), q64, kb.double(), do64, z, B, L, heads,
                                                               plan)[0]
        for pn, gp in perts.items():
            if torch.equal(gp, ref):
                continue
            r = float(((out[rc] - gp[rc]).abs() / tol[rc]).max())
            rep.call[pn] = max(rep.call.get(pn, 0.0), r)


def _masked(args, s, sc, plan, perturb=None):
    a = list(args)
    # masked_layer_bwd_ref takes one scale s for all sites: with p_attn = 0 the attention's mask is all ones, so its
    # scale must be 1; the attention stage is then run through the unmasked stage at scale 1
    if sc == 1.0:
        return _masked_hidden_only(a, s, plan, perturb)
    return D.masked_layer_bwd_ref(*a, s, perturb=perturb, plan=plan)


def _masked_hidden_only(a, s, plan, perturb):
    orig = D.masked_attention_stage

    def stage(qkv, kb, dout, edout, B, L, heads, fmt, am, s_, pt=None):
        return orig(qkv, kb, dout, edout, B, L, heads, fmt, am, 1.0, pt)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(D, "masked_attention_stage", stage)
        return D.masked_layer_bwd_ref(*a, s, perturb=perturb, plan=plan)


def _dense_rows_equal(e, ids, lens, d_out, drop, slots, row_tok, real, M, name):
    """Align 16: the dense backward of the same batch; every captured row of a real token must be its dense row, bit for
    bit (the forward is bit-identical, and d X_in is row-local: dgrad GEMMs, LayerNorm, per-sequence attention)."""
    lh = lens.to(torch.int32)
    _, ws = e.enc.forward_train(ids.to(torch.int32).cuda(), lh.cuda(), None, drop)
    _, dslots = _backward(e, ws, d_out)
    B = ids.shape[0]
    rows = torch.nonzero(real).flatten().cuda()
    toks = row_tok.cuda()[rows]
    assert torch.equal(slots[e.n_layer][:B], dslots[e.n_layer][:B]), name
    for s in range(e.n_layer):
        same = (slots[s][rows] == dslots[s][toks]).all(1)
        assert bool(same.all()), (name, "slot", s, int((~same).sum()), "rows differ from the dense backward")


# ------------------------------------------------------------------------------------------------
# batches
# ------------------------------------------------------------------------------------------------
def _batch(lens, L, seed, cls=0, pad=1):
    g = torch.Generator().manual_seed(seed)
    lens = torch.tensor(lens, dtype=torch.long)
    B = len(lens)
    keep = torch.arange(L)[None, :] < lens[:, None]
    ids = torch.where(keep, torch.randint(3, VOCAB, (B, L), generator=g), torch.full((B, L), pad, dtype=torch.long))
    ids[:, 0] = cls
    return ids, lens


def _edge_lens(L):
    return sorted({min(n, L) for n in (1, 15, 16, 17, 63, 64, 65, 127, 128, 129, L)}, reverse=True)


def _chunks(x, n):
    return [x[i:i + n] for i in range(0, len(x), n)]


def _straddles(row0, lens):
    return any(int(r) // 128 != (int(r) + int(n) - 1) // 128 for r, n in zip(row0, lens))


# ------------------------------------------------------------------------------------------------
# configurations
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
def test_packed_layers_12(gpu_lib, fmt):
    """RoBERTa + head at 12 layers, align 16: a FirstP-like passage call at 8 x 512 and a query call at 8 x 64."""
    _, e = _roberta(fmt, 12)
    e.enc.set_param("train_max_len", 512)
    rep = _Report()
    for i, (lens, L) in enumerate((([512, 1, 17, 60, 96, 128, 129, 200], 512), ([64, 1, 9, 16, 17, 33, 48, 63], 64))):
        ids, ln = _batch(lens, L, 10 + i)
        fwd = _forward(e, ids, ln, 16)
        _check_ws(e, ids, ln, fwd, _d_out(len(lens), 768, 20 + i), rep, f"12L {fmt} {len(lens)}x{L}", 16)
    rep.show(f"packed 12 layers {fmt}")
    assert rep.held.get("cls_residual_dense_rows", 0) >= 1 and "attention_whole_tile" in rep.pert


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("align", [16, 1])
def test_packed_layers_2(gpu_lib, fmt, align):
    """2 layers + head at L in {64, 128, 256, 512}, lengths at every tile and block edge (1, 15 / 16 / 17, 63 / 64 /
    65, 127 / 128 / 129, L), and a batch of 40 short sequences sharing tiles; at align 1 a plan whose sequences straddle
    tiles."""
    _, e = _roberta(fmt, 2, seed=1)
    e.enc.set_param("train_max_len", 512)
    rep = _Report()
    # the edge lengths in batches of at most 4,096 dense rows, so that the dense backward's slots are captured too
    cases = [(c, L) for L in (64, 128, 256, 512) for c in _chunks(_edge_lens(L), CAPTURE_ROWS // L)]
    g = torch.Generator().manual_seed(align)
    cases.append((torch.randint(1, 21, (40,), generator=g).tolist(), 64))
    straddle = False
    for i, (lens, L) in enumerate(cases):
        ids, ln = _batch(lens, L, 30 + i)
        fwd = _forward(e, ids, ln, align)
        _check_ws(e, ids, ln, fwd, _d_out(len(lens), 768, 40 + i), rep, f"2L {fmt} align {align} {len(lens)}x{L}", align)
        straddle |= _straddles(_pack_rows(gpu_lib, ln, L, e.enc.max_tokens, align)[0], ln)
    assert straddle or align == 16
    rep.show(f"packed 2 layers align {align} {fmt}")
    assert "attention_whole_tile" in rep.pert
    assert align == 1 or rep.held.get("cls_residual_dense_rows", 0) >= 1


@pytest.mark.parametrize("fmt", FMTS)
def test_packed_bert_no_head(gpu_lib, fmt):
    """BERT positions without a head (pad 0, eps 1e-12), hidden 768, 2 layers, at L = 256, align 16 and 1."""
    from oracle.encoder_oracle import random_roberta_state_dict as rsd
    H = 768
    sd = rsd(seed=H, n_layer=2, hidden=H, ffn=4 * H, vocab=VOCAB, max_pos=512, head=False)
    bb = _backbone(VOCAB, H, 2, 4 * H, 512, 1, 0, 1e-12)
    bb.load_state_dict({k[len("roberta."):]: v for k, v in sd.items() if k.startswith("roberta.")}, strict=True)
    e = _Enc(bb.cuda(), _lib.ANCE_ARCH_BERT, H // 64, 0, None, fmt, eps=1e-12)
    e.enc.set_param("train_max_len", 256)
    rep = _Report()
    for align in (16, 1):
        ids, ln = _batch([256, 1, 100, 129, 16, 200, 37], 256, 60 + align, cls=101 % VOCAB, pad=0)
        fwd = _forward(e, ids, ln, align)
        _check_ws(e, ids, ln, fwd, _d_out(len(ln), H, 61 + align), rep, f"bert {fmt} align {align}", align)
    rep.show(f"packed bert no head {fmt}")


@pytest.mark.parametrize("fmt", FMTS)
def test_packed_layers_dropout(gpu_lib, fmt):
    """p_hidden = p_attn = 0.1 at align 16, L = 128 and 512; p_hidden = 0.1 alone at align 1 (the packed forward refuses
    attention dropout there), L = 128."""
    _, e = _roberta(fmt, 2, seed=3)
    e.enc.set_param("train_max_len", 512)
    rep = _Report()
    cases = [(16, _edge_lens(128) + [5, 40], 128, (P, P, 0xD0D0)), (16, [512, 200, 129, 17, 1], 512, (P, P, 0xD0D1)),
             (1, _edge_lens(128) + [5, 40, 90], 128, (P, 0.0, 0xD0D2))]
    for i, (align, lens, L, drop) in enumerate(cases):
        ids, ln = _batch(lens, L, 70 + i)
        fwd = _forward(e, ids, ln, align, drop)
        _check_ws(e, ids, ln, fwd, _d_out(len(lens), 768, 80 + i), rep, f"dropout {fmt} align {align} {len(lens)}x{L}",
                  align, drop)
    rep.show(f"packed dropout {fmt}")
    assert "attn_mask_from_tile" in rep.pert and rep.held.get("cls_residual_dense_rows", 0) >= 1


@pytest.mark.parametrize("fmt", FMTS)
def test_plan_held_in_the_workspace(gpu_lib, fmt):
    """Three packed forwards (align 16, then 1, then 16, different batches) before their backwards in reverse order: each
    backward reads its own plan from its workspace, not the handle's last one."""
    _, e = _roberta(fmt, 2, seed=4)
    rep = _Report()
    calls = [(16, _edge_lens(128), 128), (1, [100, 3, 128, 77, 64, 1, 120], 128), (16, [64, 1, 33, 17, 50], 64)]
    done = []
    for i, (align, lens, L) in enumerate(calls):
        ids, ln = _batch(lens, L, 90 + i)
        done.append((align, ids, ln, _forward(e, ids, ln, align)))
    for i, (align, ids, ln, fwd) in reversed(list(enumerate(done))):
        _check_ws(e, ids, ln, fwd, _d_out(len(ln), 768, 95 + i), rep, f"held {fmt} call {i} align {align}", align,
                  dense_equal=False)
    rep.show(f"plan held in the workspace {fmt}")


def test_layout_hook(gpu_lib):
    """ance_dbg_train_layout_packed refuses what the packed training plan refuses, with the same messages, and its total
    is ance_encoder_train_workspace_packed's at both alignments."""
    _, e = _roberta("fp16", 1)
    lib, h = e.enc.lib, e.enc.h
    out = (C.c_size_t * 24)()
    n = C.c_int()
    ok = torch.tensor([64, 1, 30, 17], dtype=torch.int32)
    for align in (16, 1):
        e.enc.set_param("varlen_align", align)
        assert lib.ance_dbg_train_layout_packed(h, ok.data_ptr(), 4, 64, out, C.byref(n)) == 0
        tot = C.c_size_t()
        assert lib.ance_encoder_train_workspace_packed(h, ok.data_ptr(), 4, 64, C.byref(tot)) == 0
        assert out[23] == tot.value and n.value >= 1
        f = dict(zip(_lib.TRAIN_LAYOUT_FIELDS, out[:15]))
        assert f["total"] == out[15] and out[15] < out[16] < out[23]   # the plan follows the train layout
    assert lib.ance_dbg_train_layout_packed(h, None, 4, 64, out, C.byref(n)) == 1
    for bad, L, msg in (([0, 10], 64, b"outside [1, 64]"), ([10, 65], 64, b"outside [1, 64]"),
                        ([200, 10], 256, b"train_max_len")):
        lh = torch.tensor(bad, dtype=torch.int32)
        assert lib.ance_dbg_train_layout_packed(h, lh.data_ptr(), 2, L, out, C.byref(n)) != 0
        assert msg in lib.ance_last_error(), lib.ance_last_error()
    big = torch.full((200,), 128, dtype=torch.int32)   # 25,600 rows: more than one plan of max_tokens 8192
    assert lib.ance_dbg_train_layout_packed(h, big.data_ptr(), 200, 128, out, C.byref(n)) != 0
    assert b"does not fit one plan" in lib.ance_last_error()
