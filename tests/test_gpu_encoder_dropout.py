"""Dropout of the trainable encoder on the GPU: the device generator bit for bit, the masks the forward applied read back
from the training workspace, identities with dropout off, and whole-model gradients against fp32 autograd of the oracle
given the same masks (tests/encoder_dropout_refs.py)."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from ance_b200 import _lib
from ance_b200.models import BiEncoder, RobertaDot_NLL_LN, _param_groups
from ance_b200.synthetic import random_roberta_state_dict, roberta_base_config
from oracle.encoder_oracle import EncoderOracle, RobertaDotOracle
from tests import encoder_dropout_refs as D
from tests import encoder_layer_refs as LR
from tests.test_gpu_encoder_backward import VOCAB, _batch, _compare_grads, _model
from tests.test_gpu_encoder_backward_layers import GATE_12, _rel
from tests.test_gpu_encoder_backward_layers import _batch as lbatch
from tests.test_gpu_encoder_backward_layers import _d_out
from tests.test_gpu_encoder_backward_layers import _roberta as lroberta
from tests.test_gpu_encoder_backward_long import _maxp

pytestmark = pytest.mark.gpu

FMTS = ["fp16", "bf16"]
FMT_CODE = {"fp16": _lib.ANCE_FMT_FP16, "bf16": _lib.ANCE_FMT_BF16}
U16 = {"fp16": 2.0 ** -11, "bf16": 2.0 ** -8}
P = 0.1


@pytest.fixture(scope="module")
def gpu_lib():
    assert torch.cuda.is_available()
    return _lib.load()


def test_generator_matches_numpy(gpu_lib):
    """ance_dbg_dropout_bits against the numpy Philox4x32-10: 2.6 M calls (10.5 M words) across a carry of the counter's
    low word, with every counter and key word nonzero."""
    n = 2_621_440
    for seed, sw, first in ((0x0123456789ABCDEF, 0xDEADBEEF00C0FFEE, 0xFFFFFFFF - 1_000_000), (0, 7, 0)):
        out = torch.empty(4 * n, dtype=torch.int32, device="cuda")
        _lib.check(gpu_lib.ance_dbg_dropout_bits(seed, sw, first, n, out.data_ptr(), _lib.current_stream()))
        got = out.cpu().numpy().view(np.uint32)
        assert np.array_equal(got, D.dbg_bits(seed, sw, first, n))


def _layout(enc, B, L):
    lo = (C.c_size_t * len(_lib.TRAIN_LAYOUT_FIELDS))()
    _lib.check(enc.lib.ance_dbg_train_layout(enc.h, B, L, lo))
    return dict(zip(_lib.TRAIN_LAYOUT_FIELDS, list(lo)))


def _slot(ws, lay, off, rows, cols, fmt, layer=None):
    base = off if layer is None else lay["layers"] + layer * lay["per_layer"] + off
    raw = ws[base:base + rows * cols * 2].view(torch.bfloat16 if fmt == "bf16" else torch.float16)
    return raw.view(rows, cols).double().cpu()


def _written(ws, lay, B, L, n_layer, H=768, F=3072):
    """The bytes of a training workspace the forward writes (slot padding and the unused rows of the pruned last layer's
    compact slots are left as allocated)."""
    M = B * L
    parts = [ws[lay["ids"]:lay["ids"] + 4 * M], ws[lay["kbias"]:lay["kbias"] + 4 * M]]
    for l in range(n_layer):
        base = lay["layers"] + l * lay["per_layer"]
        rows = B if l == n_layer - 1 else M
        for f, n in (("x_in", M * H), ("qkv", M * 3 * H), ("ctx", M * H), ("t1", rows * H), ("x1", rows * H),
                     ("u", rows * F), ("ff", rows * F), ("t2", rows * H)):
            parts.append(ws[base + lay[f]:base + lay[f] + 2 * n])
    parts += [ws[lay["x_final"]:lay["x_final"] + 2 * B * H], ws[lay["head_in"]:lay["head_in"] + 4 * B * H]]
    return torch.cat(parts)


def _grads(enc, model, d_out, ws):
    groups = _param_groups(model.roberta, (model.embeddingHead, model.norm))
    flat = [torch.empty_like(t) for t in groups[0] + [x for l in groups[1] for x in l] + groups[2]]
    n = len(groups[1])
    g = (flat[:5], [flat[5 + 16 * i:5 + 16 * (i + 1)] for i in range(n)], flat[5 + 16 * n:])
    enc.backward(d_out, ws, g)
    torch.cuda.synchronize()
    return flat


@pytest.mark.parametrize("fmt", FMTS)
def test_p0_and_repeated_seed_are_identities(gpu_lib, fmt):
    """p = 0 through the dropout entry point is ance_encoder_forward_train: output and every saved activation equal, and
    every gradient bit-identical except the scatter-added word / position rows.  The same holds for two calls with the
    same seed at p = 0.1."""
    m, _ = _model(fmt)
    enc = m._encoder(torch.device("cuda"))
    enc.set_param("train_max_len", 512)
    enc.update_weights(m.roberta, (m.embeddingHead, m.norm))
    for L in (64, 256):
        ids, mask = _batch(3, L, L, holed=True)
        i32, m8 = ids.to(torch.int32).cuda(), mask.to(torch.uint8).cuda()
        d_out = torch.randn(3, 768, generator=torch.Generator().manual_seed(L)).cuda()
        for a_args, b_args in ((None, (0.0, 0.0, 99)), ((P, P, 1234), (P, P, 1234))):
            oa, wa = enc.forward_train(i32, None, m8, a_args)
            ob, wb = enc.forward_train(i32, None, m8, b_args)
            lay = _layout(enc, 3, L)
            assert torch.equal(oa, ob), (L, a_args)
            assert torch.equal(_written(wa, lay, 3, L, 2), _written(wb, lay, 3, L, 2)), (L, a_args)
            ga, gb = _grads(enc, m, d_out, wa), _grads(enc, m, d_out, wb)
            for i, (x, y) in enumerate(zip(ga, gb)):
                if i in (0, 1):   # word / position rows: fp32 atomics, order varies
                    torch.testing.assert_close(x, y, rtol=1e-5, atol=1e-6)
                else:
                    assert torch.equal(x, y), (L, a_args, i)
    with pytest.raises(_lib.AnceError, match=r"\[0, 1\)"):
        enc.forward_train(i32, None, m8, (1.0, 0.0, 1))
    with pytest.raises(_lib.AnceError, match=r"\[0, 1\)"):
        enc.forward_train(i32, None, m8, (0.0, float("nan"), 1))


def test_eval_no_grad_and_seeds(gpu_lib):
    """dropout=True under eval(), or without grad, is dropout off; torch.manual_seed reproduces a step; another seed
    changes the embeddings."""
    m, _ = _model("fp16")
    ids, mask = _batch(4, 128, 5)
    q = (ids.cuda(), mask.cuda())
    m.set_trainable(True)
    ref = m.query_emb(*q).detach()
    m.set_trainable(True, dropout=True)
    assert m._dropout == (0.1, 0.1)
    m.eval()
    assert torch.equal(m.query_emb(*q).detach(), ref)
    m.train()
    with torch.no_grad():
        assert torch.equal(m.query_emb(*q), ref)
    w = torch.randn(4, 768, generator=torch.Generator().manual_seed(1)).cuda()
    runs = []
    for s in (7, 7, 8):
        m.zero_grad()
        torch.manual_seed(s)
        e = m.query_emb(*q)
        (e * w).sum().backward()
        runs.append((e.detach().clone(), [p.grad.clone() for p in m.parameters()]))
    assert not torch.equal(runs[0][0], ref)
    assert torch.equal(runs[0][0], runs[1][0])
    for i, (x, y) in enumerate(zip(runs[0][1], runs[1][1])):
        if i in (0, 1):
            torch.testing.assert_close(x, y, rtol=1e-5, atol=1e-6)
        else:
            assert torch.equal(x, y), i
    assert not torch.equal(runs[0][0], runs[2][0])


# ------------------------------------------------------------------------------------------------
# the forward, stage by stage, from the workspace
# ------------------------------------------------------------------------------------------------
def _w16(t, fmt):
    return t.detach().to(torch.bfloat16 if fmt == "bf16" else torch.float16).double().cpu()


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("L", [8, 64, 128, 256, 512])
def test_forward_stages_from_the_workspace(gpu_lib, fmt, L):
    """X0, CTX, T1 and T2 of both layers (T1 / T2 of the pruned last layer: the CLS rows) against fp64 of the saved
    inputs with the numpy masks.  Bounds: the 16-bit rounding of the stored result and of the 16-bit operands it was
    formed from; the wrong-mask perturbations (another seed, the attention mask transposed, the last layer's rows
    taken as tokens 0..B-1) fall outside."""
    m, _ = _model(fmt)
    enc = m._encoder(torch.device("cuda"))
    enc.set_param("train_max_len", 512)
    enc.update_weights(m.roberta, (m.embeddingHead, m.norm))
    B = max(2, min(6, 1024 // L))
    ids, mask = _batch(B, L, 300 + L, holed=L != 8)
    if B > 2:
        ids[2, 1:] = 1
        mask[2, 1:] = 0   # a sequence of padding only
    seed = 0x5EED0000 + L
    i32, m8 = ids.to(torch.int32).cuda(), mask.to(torch.uint8).cuda()
    _, w0 = enc.forward_train(i32, None, m8)
    _, wd = enc.forward_train(i32, None, m8, (P, P, seed))
    torch.cuda.synchronize()
    lay = _layout(enc, B, L)
    M, H, u = B * L, 768, U16[fmt]
    s = D.scale(P)

    def check(name, got, ref, tol, perts):
        err = float(((got - ref).abs() / tol).max())
        assert err <= 1.0, (name, err)
        for pn, pr in perts.items():
            assert float(((got - pr).abs() / tol).max()) > 1.0, (name, pn)

    # X0 = m o LN(E) s: the unmasked LN output from the run without dropout
    x0 = _slot(wd, lay, lay["x_in"], M, H, fmt, 0)
    x0n = _slot(w0, lay, lay["x_in"], M, H, fmt, 0)
    hm = torch.tensor(D.hidden_mask(seed, D.SITE_EMBED, 0, np.arange(M), H, P))
    tol = 3 * u * x0n.abs() * s + 1e-7
    check("X0", x0, x0n * hm * s, tol,
          {"another seed": x0n * torch.tensor(D.hidden_mask(seed + 1, D.SITE_EMBED, 0, np.arange(M), H, P)) * s})
    kb = (wd[lay["kbias"]:lay["kbias"] + 4 * M].view(torch.float32).double().cpu() / np.log2(np.e)).numpy()
    layers = m.roberta.encoder.layer
    for l in range(2):
        last = l == 1
        x_in = _slot(wd, lay, lay["x_in"], M, H, fmt, l)
        qkv = _slot(wd, lay, lay["qkv"], M, 3 * H, fmt, l).numpy()
        ctx = _slot(wd, lay, lay["ctx"], M, H, fmt, l)
        ref, bnd, tr = np.zeros((M, H)), np.zeros((M, H)), np.zeros((M, H))
        for b in range(B):
            rows = slice(b * L, (b + 1) * L)
            for h in range(12):
                q, k, v = (qkv[rows, c * H + h * 64:c * H + h * 64 + 64] for c in range(3))
                am = D.attn_mask(seed, l, b, h, 12, L, P)
                o, pr = D.attention_fwd(q, k, v, kb[rows], am, s)
                ref[rows, h * 64:h * 64 + 64] = o
                bnd[rows, h * 64:h * 64 + 64] = (pr * am * s) @ np.abs(v)
                tr[rows, h * 64:h * 64 + 64] = D.attention_fwd(q, k, v, kb[rows], am.T, s)[0]
        tol = torch.tensor(2 * u * bnd + 2 * u * np.abs(ref) + 1e-6)
        check(f"CTX layer {l}", ctx, torch.tensor(ref), tol, {"attention mask indexed (j, i)": torch.tensor(tr)})
        # T1 = m o (CTX Wo^T + bo) s + X_in ; T2 = m o (FF W2^T + b2) s + X1  (last layer: compact CLS rows)
        toks = np.arange(B) * L if last else np.arange(M)
        rows = torch.tensor(toks)
        n = len(toks)
        lw = layers[l]
        for site, a_in, w_, b_, res, slot in (
                (D.SITE_ATTN_OUT, ctx[rows], lw.attention.output.dense.weight, lw.attention.output.dense.bias, x_in[rows], "t1"),
                (D.SITE_FFN_OUT, _slot(wd, lay, lay["ff"], n, 3072, fmt, l), lw.output.dense.weight, lw.output.dense.bias,
                 _slot(wd, lay, lay["x1"], n, H, fmt, l), "t2")):
            W = _w16(w_, fmt)
            br = a_in @ W.T + b_.detach().double().cpu()
            mk = torch.tensor(D.hidden_mask(seed, site, l, toks, H, P))
            got = _slot(wd, lay, lay[slot], n, H, fmt, l)
            ref = br * mk * s + res
            tol = 2 * u * ref.abs() + 1e-4 * (a_in.abs() @ W.abs().T) * s + 1e-6
            perts = {"mask of another layer": br * torch.tensor(D.hidden_mask(seed, site, 1 - l, toks, H, P)) * s + res}
            if last:
                perts["CLS rows as tokens 0..B-1"] = br * torch.tensor(D.hidden_mask(seed, site, l, np.arange(n), H, P)) * s + res
            check(f"{slot} layer {l}", got, ref, tol, perts)


# ------------------------------------------------------------------------------------------------
# whole model against the oracle with the same masks
# ------------------------------------------------------------------------------------------------
def _seeds(torch_seed, n):
    """The mask seeds the model draws for its next n trainable encodes after torch.manual_seed(torch_seed)."""
    torch.manual_seed(torch_seed)
    out = []
    for _ in range(n):
        lo, hi = torch.randint(0, 2 ** 32, (2,), dtype=torch.int64).tolist()
        out.append(lo | (hi << 32))
    torch.manual_seed(torch_seed)
    return out


def _masked_oracle_loss(sd, batches, seeds, objective, n_layer=2):
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        orc = RobertaDotOracle(sd, n_layer=n_layer, device="cuda")
        leaves = {k: v.detach().clone().requires_grad_(True) for k, v in orc.enc.sd.items()}
        orc.enc.sd = leaves
        hw, hb, ng, nb = (t.detach().clone().requires_grad_(True) for t in (orc.head_w, orc.head_b, orc.norm_g, orc.norm_b))
        embs = [Fn.layer_norm(Fn.linear(D.masked_hidden_states(orc.enc, i, k, sd_, P, P)[:, 0], hw, hb), (768,), ng, nb, 1e-5)
                for (i, k), sd_ in zip(batches, seeds)]
        out = objective(*embs)
        out.backward()
        grads = {k: v.grad for k, v in leaves.items()}
        grads.update({"embeddingHead.weight": hw.grad, "embeddingHead.bias": hb.grad, "norm.weight": ng.grad,
                      "norm.bias": nb.grad})
        grads["roberta.embeddings.word_embeddings.weight"][1] = 0
        grads["roberta.embeddings.position_embeddings.weight"][1] = 0
        return float(out.detach()), grads
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("kind", ["psg", "firstp"])
def test_roberta_gradients_match_the_masked_oracle(gpu_lib, fmt, kind):
    """rdot_nll passages (64-token queries, 128-token passages) and FirstP (512-token documents), p = 0.1 at every site,
    every parameter gradient under the existing gates against the oracle run with the same masks."""
    m, sd = _model(fmt)
    m.train()
    Ld = 128 if kind == "psg" else 512
    m.set_trainable(True, max_len=max(128, Ld), dropout=True)
    q, a, b = _batch(4, 64, 41), _batch(4, Ld, 42, holed=True), _batch(4, Ld, 43)
    w = torch.randn(3, 4, 768, generator=torch.Generator().manual_seed(44)).cuda()

    def objective(eq, ea, eb):
        lm = torch.stack([(eq * ea).sum(-1), (eq * eb).sum(-1)], dim=1)
        return (-torch.log_softmax(lm, dim=1)[:, 0]).mean() + (eq * w[0]).sum() + (ea * w[1]).sum() + (eb * w[2]).sum()

    seeds = _seeds(100 + Ld, 3)
    loss = objective(m.query_emb(q[0].cuda(), q[1].cuda()), m.body_emb(a[0].cuda(), a[1].cuda()),
                     m.body_emb(b[0].cuda(), b[1].cuda()))
    loss.backward()
    _, gref = _masked_oracle_loss(sd, [q, a, b], seeds, objective)
    _compare_grads(m, gref, fmt, f"{kind} dropout {P}")
    # the oracle with the masks of other seeds is far from these gradients: which mask was applied matters at this gate
    _, g0 = _masked_oracle_loss(sd, [q, a, b], [seeds[0] + 1, seeds[1] + 1, seeds[2] + 1], objective)
    k = "roberta.encoder.layer.0.attention.output.dense.weight"
    assert float((m.roberta.encoder.layer[0].attention.output.dense.weight.grad - g0[k]).norm() / g0[k].norm()) > 0.05


@pytest.mark.parametrize("fmt", FMTS)
def test_biencoder_gradients_match_the_masked_oracle(gpu_lib, fmt):
    """DPR at 256 tokens, dropout=True (0.1 / 0.1), triplet loss plus fixed-weight terms, against the masked oracle."""
    sd = {**random_roberta_state_dict(seed=61, n_layer=2, vocab=VOCAB, max_pos=512, head=False, prefix="question_model."),
          **random_roberta_state_dict(seed=62, n_layer=2, vocab=VOCAB, max_pos=512, head=False, prefix="ctx_model.")}
    m = BiEncoder(type("A", (), {"num_hidden_layers": 2, "vocab_size": VOCAB})())
    m.load_state_dict(sd)
    m = m.cuda()
    m.encoder_operand = fmt
    m.set_trainable(True, max_len=256, dropout=True)
    assert m._dropout == (0.1, 0.1)

    def bert_batch(B, seed):
        ids, mask = _batch(B, 256, seed)
        ids = torch.where(mask.bool(), ids, torch.zeros_like(ids))
        ids[:, 0] = 101
        return ids, mask

    q, a, b = bert_batch(4, 71), bert_batch(4, 72), bert_batch(4, 73)
    w = torch.randn(3, 4, 768, generator=torch.Generator().manual_seed(74)).cuda() * 0.05

    def objective(eq, ea, eb):
        lm = torch.stack([(eq * ea).sum(-1), (eq * eb).sum(-1)], dim=1)
        return (-torch.log_softmax(lm, dim=1)[:, 0]).mean() + (eq * w[0]).sum() + (ea * w[1]).sum() + (eb * w[2]).sum()

    seeds = _seeds(5, 3)
    qe, ae, be = m.query_emb(q[0].cuda(), q[1].cuda()), m.body_emb(a[0].cuda(), a[1].cuda()), m.body_emb(b[0].cuda(), b[1].cuda())
    loss = objective(qe, ae, be)
    loss.backward()
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        orc = [EncoderOracle(sd, p, "bert", 2, 12, 0, 1e-12, device="cuda") for p in ("question_model.", "ctx_model.")]
        for o in orc:
            o.sd = {k: v.detach().clone().requires_grad_(True) for k, v in o.sd.items()}
        embs = [D.masked_hidden_states(o, x[0], x[1], s_, P, P)[:, 0] for o, x, s_ in zip((orc[0], orc[1], orc[1]), (q, a, b), seeds)]
        out = objective(*embs)
        out.backward()
        gref = {}
        for o in orc:
            for k, v in o.sd.items():
                gref[k] = v.grad if v.grad is not None else torch.zeros_like(v)
            gref[o.p + "embeddings.word_embeddings.weight"][0] = 0
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
    assert abs(float(loss) - float(out)) <= 0.02 * abs(float(out)), (float(loss), float(out))
    _compare_grads(m, gref, fmt, f"BiEncoder dropout {P}")


# ------------------------------------------------------------------------------------------------
# the backward, layer by layer, with the masked mirror
# ------------------------------------------------------------------------------------------------
DT16 = {"fp16": torch.float16, "bf16": torch.bfloat16}


def _check_call_dropout(e, ids, mask, d_out, seed, worst, name):
    """One dropout forward_train + backward on the capture handle `e` (tests/test_gpu_encoder_backward_layers._Enc):
    every stage of every layer against tests/encoder_dropout_refs.masked_layer_bwd_ref on the kernel's own activations
    and captured upstream gradients, the embedding stage on m o dX0 s; each perturbation of the dropout rules must put
    some gradient of the call outside the bound."""
    B, L = ids.shape
    M, H, fmt, NL, heads = B * L, e.H, e.fmt, e.n_layer, e.heads
    _, ws = e.enc.forward_train(ids.to(torch.int32).cuda(), None, mask.to(torch.uint8).cuda(), (P, P, seed))
    embs, layers, hd = e.groups
    mk = lambda ts: [torch.full(t.shape, float("nan"), device="cuda") for t in ts]
    grads = (mk(embs), [mk(l) for l in layers], mk(hd))
    e.enc.backward(d_out, ws, grads)
    slots = []
    for sl in range(NL + 1):
        buf = torch.empty(4096, H, device="cuda")
        _lib.check(e.enc.lib.ance_encoder_debug_grads(e.enc.h, sl, buf.data_ptr(), _lib.current_stream()))
        slots.append(buf)
    torch.cuda.synchronize()
    lo = e.layout(B, L)
    a16 = lambda off, rows, cols: ws[off:off + rows * cols * 2].view(DT16[fmt]).view(rows, cols).to(torch.float64)
    kb = ws[lo["kbias"]:lo["kbias"] + M * 4].view(torch.float32).to(torch.float64)
    gembs, glayers, ghd = grads
    s = D.scale(P)
    rejected = {n: 0.0 for n in D.PERTURBATIONS + ("embedding mask not applied",)}

    def record(stage, out, g, t, perts):
        for k in g:
            err = float(((out[k].double() - g[k]).abs() / t[k]).max())
            assert err <= 1.0, (name, stage, k, err)
            worst[stage] = max(worst.get(stage, 0.0), err)
        for pn, gp in perts.items():
            rejected[pn] = max(rejected[pn], max(float(((out[k].double() - gp[k]).abs() / t[k]).max()) for k in g))

    x_final = a16(lo["x_final"], B, H)
    head_in = ws[lo["head_in"]:lo["head_in"] + B * H * 4].view(torch.float32).view(B, H).to(torch.float64)
    g, t = LR.head_bwd_ref(d_out, head_in, x_final, _w16(hd[0], fmt).cuda(), hd[2].detach())
    record("head", dict(zip(LR.HEAD_GRADS, ghd), x_final=slots[NL][:B]), g, t, {})
    for l in reversed(range(NL)):
        last = l == NL - 1
        Mr = B if last else M
        base = lo["layers"] + l * lo["per_layer"]
        F = layers[l][10].shape[0]
        act = {"x_in": a16(base + lo["x_in"], M, H), "qkv": a16(base + lo["qkv"], M, 3 * H),
               "ctx": a16(base + lo["ctx"], M, H), "t1": a16(base + lo["t1"], Mr, H), "x1": a16(base + lo["x1"], Mr, H),
               "u": a16(base + lo["u"], Mr, F), "ff": a16(base + lo["ff"], Mr, F), "t2": a16(base + lo["t2"], Mr, H)}
        p = layers[l]
        w = {"wqkv": _w16(torch.cat([p[0], p[2], p[4]]), fmt).cuda(), "wo": _w16(p[6], fmt).cuda(),
             "w1": _w16(p[10], fmt).cuda(), "w2": _w16(p[12], fmt).cuda(), "ln1_g": p[8].detach(), "ln2_g": p[14].detach()}
        toks = np.arange(B) * L if last else np.arange(M)
        hm = [torch.tensor(D.hidden_mask(seed, site, l, toks, H, P), device="cuda") for site in (D.SITE_ATTN_OUT, D.SITE_FFN_OUT)]
        am = torch.tensor(D.attn_masks(seed, l, B, heads, L, P), device="cuda")
        dy = slots[l + 1][:Mr]
        args = (act, kb, w, dy, B, L, heads, last, e.eps, fmt, hm[0], hm[1], am, s)
        g, t = D.masked_layer_bwd_ref(*args)
        perts = {n: D.masked_layer_bwd_ref(*args, perturb=n)[0] for n in D.PERTURBATIONS}
        record("layer", dict(zip(LR.LAYER_GRADS, glayers[l]), x_in=slots[l][:M]), g, t, perts)
    # embeddings: the LayerNorm gets m o dX0 s, formed in fp32 as the kernel forms it
    m0 = torch.tensor(D.hidden_mask(seed, D.SITE_EMBED, 0, np.arange(M), H, P), dtype=torch.float32, device="cuda")
    dx0 = slots[0][:M]
    dx0m = (dx0 * torch.tensor(s, dtype=torch.float32)) * m0
    eargs = [x.detach() for x in embs[:4]]
    g, t = LR.embedding_stage_ref(ids.cuda(), dx0m, *eargs, e.eps, e.pad, e.roberta)
    gp, _ = LR.embedding_stage_ref(ids.cuda(), dx0, *eargs, e.eps, e.pad, e.roberta)
    record("embeddings", dict(zip(("word_emb", "pos_emb", "type_emb", "emb_ln_g", "emb_ln_b"), gembs)), g, t,
           {"embedding mask not applied": gp})
    print(f"{name}: perturbed err / bound {({k: round(v, 2) for k, v in rejected.items()})}")
    for pn, v in rejected.items():
        assert v > 1.0 or pn in ATTN_ONLY, (name, pn, v)


# Perturbations confined to the attention backward's inner arithmetic: through a layer, on random weights, they stay
# inside the attention stage's propagated bound (as the unmasked mirror's "qk_bias_swap" does); they are asserted on the
# kernel itself, test_attention_backward_dropout_kernel, and printed here.
ATTN_ONLY = ("d_unmasked", "mask_transposed")


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("L", [64, 128, 256, 512])
def test_attention_backward_dropout_kernel(gpu_lib, fmt, L):
    """The attention backward with dropout (ance_dbg_attention_backward_dropout: attn_bwd_kernel<., true> for L <= 128,
    dq_kernel / dkv_kernel<., true> above) against the masked fp64 reference, under the unmasked kernel's bound times s
    (encoder_dropout_refs.masked_attention_stage's argument); every perturbation of the dropout rules rejected."""
    from tests import encoder_grad_long_refs as R
    from tests import encoder_grad_refs as G
    B, heads = max(2, 1024 // L), 3
    H = heads * 64
    s = D.scale(P)
    for cls_only in (0, 1):
        qkv, kb, dout, dfull = R.inputs(B, L, heads, fmt, ["full", "holed", "prefix", "allpad"], L + cls_only, cls_only)
        dqkv = torch.empty(B * L, 3 * H, device="cuda")
        seed, layer = 0xA77 + L, 3
        qd, kd, dd = qkv.cuda(), kb.cuda(), dout.cuda()
        _lib.check(gpu_lib.ance_dbg_attention_backward_dropout(FMT_CODE[fmt], qd.data_ptr(), kd.data_ptr(), dd.data_ptr(),
                                                               cls_only, B, L, heads, P, seed, layer, dqkv.data_ptr(),
                                                               _lib.current_stream()))
        torch.cuda.synchronize()
        am = torch.tensor(D.attn_masks(seed, layer, B, heads, L, P))
        ref = D.masked_attention_bwd_ref(qkv, kb, dfull, B, L, heads, am, s)
        tol = (G.attention_bwd_tol(qkv, kb, dfull, B, L, heads) if L <= 128 else
               R.attention_bwd_long_tol(qkv, kb, dfull, B, L, heads, fmt)) * s * (1 + 4 * 2.0 ** -24)
        out = dqkv.cpu().double()
        err = float(((out - ref).abs() / tol).max())
        perts = {n: float(((out - D.masked_attention_bwd_ref(qkv, kb, dfull, B, L, heads, am, s, n)).abs() / tol).max())
                 for n in ("no_mask_bwd", "no_scale_bwd", "d_unmasked", "mask_transposed")}
        print(f"attn bwd dropout {fmt} L{L} cls{cls_only}: err / bound {err:.3f}; perturbed {({k: round(v, 2) for k, v in perts.items()})}")
        assert err <= 1.0, (L, cls_only, err)
        for n, v in perts.items():
            assert v > 1.0, (L, cls_only, n, v)


@pytest.mark.parametrize("fmt", FMTS)
def test_layers_12_bench_shape_dropout(gpu_lib, fmt):
    """12 layers + head at the bench shape (8 x 64, 8 x 128, 8 x 128), p = 0.1 at every site."""
    _, e = lroberta(fmt, 12)
    worst = {}
    for i, (B, L) in enumerate(((8, 64), (8, 128), (8, 128))):
        ids, mask = lbatch(B, L, 100 + i)
        _check_call_dropout(e, ids, mask, _d_out(B, 768, i), 0xD00D + i, worst, f"12L {fmt} {B}x{L}")
    print(f"12 layers dropout {fmt}: worst err / bound {({k: round(v, 3) for k, v in worst.items()})}")


@pytest.mark.parametrize("fmt", FMTS)
def test_layers_long_dropout(gpu_lib, fmt):
    """2 layers + head at 3 x 256 and 2 x 512 (holed masks, a length-1 sequence), p = 0.1 at every site."""
    _, e = lroberta(fmt, 2, seed=5)
    e.enc.set_param("train_max_len", 512)
    worst = {}
    for i, (B, L) in enumerate(((3, 256), (2, 512))):
        ids, mask = lbatch(B, L, 700 + i)
        _check_call_dropout(e, ids, mask, _d_out(B, 768, 70 + i), 0xBEEF + i, worst, f"2L {fmt} {B}x{L}")
    print(f"long layers dropout {fmt}: worst err / bound {({k: round(v, 3) for k, v in worst.items()})}")


# ------------------------------------------------------------------------------------------------
# MaxP, 12-layer FirstP and an SGD trajectory with dropout
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
def test_maxp_gradients_match_the_masked_oracle(gpu_lib, fmt):
    """MaxP: 2 documents x 4 chunks of 512 (one chunk all padding), one mask seed for the 8 chunks of the call."""
    from ance_b200.models import RobertaDot_CLF_ANN_NLL_MultiChunk
    _, sd = _model(fmt)
    m = RobertaDot_CLF_ANN_NLL_MultiChunk(roberta_base_config(num_hidden_layers=2, vocab_size=VOCAB))
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    m.encoder_operand = fmt
    m.set_trainable(True, max_len=512, dropout=True)
    g = torch.Generator().manual_seed(51)
    ids = torch.randint(3, VOCAB, (2, 2048), generator=g)
    ids[:, ::512] = 0
    lens = torch.tensor([2048, 1300])
    mask = (torch.arange(2048)[None, :] < lens[:, None]).to(torch.int64)
    ids = torch.where(mask.bool(), ids, torch.ones_like(ids))
    qv = torch.randn(768, generator=g).cuda()
    seeds = _seeds(52, 1)
    emb = m.body_emb(ids.cuda(), mask.cuda())
    _maxp(emb, qv.expand(2, 768), mask.cuda()).max(-1).values.sum().backward()

    def objective(ex):
        return _maxp(ex.reshape(2, 4, 768), qv.expand(2, 768), mask.cuda()).max(-1).values.sum()

    _, gref = _masked_oracle_loss(sd, [(ids.reshape(8, 512), mask.reshape(8, 512))], seeds, objective)
    _compare_grads(m, gref, fmt, f"MaxP dropout {P}")


@pytest.mark.parametrize("fmt", FMTS)
def test_firstp_twelve_layers_dropout(gpu_lib, fmt):
    """12-layer FirstP (4 queries x 64, 2 + 2 documents x 512) with dropout, under the 12-layer rule: GATE_12 plus twice
    the measured effect of the forward's 16-bit storage, both references given the same masks."""
    sd = random_roberta_state_dict(seed=0, n_layer=12, vocab=VOCAB)
    m = RobertaDot_NLL_LN(roberta_base_config(num_hidden_layers=12, vocab_size=VOCAB))
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    m.encoder_operand = fmt
    m.set_trainable(True, max_len=512, dropout=True)
    batches = [_batch(4, 64, 81), _batch(2, 512, 82), _batch(2, 512, 83, holed=True)]
    w = [torch.randn(b[0].shape[0], 768, generator=torch.Generator().manual_seed(84 + i)).cuda() for i, b in enumerate(batches)]

    def objective(*es):
        return sum((e_ * w_).sum() for e_, w_ in zip(es, w))

    seeds = _seeds(85, 3)
    objective(*[m.body_emb(i.cuda(), k.cuda()) for i, k in batches]).backward()
    _, ref = D.masked_autograd_grads(sd, batches, seeds, objective, P, P)
    _, rnd = D.masked_autograd_grads(sd, batches, seeds, objective, P, P, fmt)
    bad, ratios = [], {}
    for k, p in m.state_dict(keep_vars=True).items():
        gate = GATE_12[fmt] + 2 * _rel(rnd[k], ref[k], k, ref)
        ratios[k] = _rel(p.grad, ref[k], k, ref) / gate
        if not ratios[k] <= 1.0:
            bad.append((k, ratios[k]))
    top = sorted(ratios, key=ratios.get, reverse=True)[:3]
    print(f"12 layers FirstP dropout {fmt}: relative error / gate, largest: " + ", ".join(f"{k} {ratios[k]:.3f}" for k in top))
    assert not bad, bad


def test_firstp_sgd_trajectory_dropout(gpu_lib):
    """20 SGD steps of FirstP (4 triplets at (64, 512, 512), lr 0.05) with dropout, fresh masks every step: each step's
    loss within 0.02 of the oracle's trajectory given the same masks."""
    m, sd = _model("fp16", seed=3)
    m.set_trainable(True, max_len=512, dropout=True)
    q, a, b = _batch(4, 64, 91), _batch(4, 512, 92), _batch(4, 512, 93)
    lr = 0.05
    opt = torch.optim.SGD(m.parameters(), lr=lr)

    def nll(eq, ea, eb):
        lm = torch.stack([(eq * ea).sum(-1), (eq * eb).sum(-1)], dim=1)
        return (-torch.log_softmax(lm, dim=1)[:, 0]).mean()

    ours, step_seeds = [], []
    for i in range(20):
        step_seeds.append(_seeds(2000 + i, 3))
        opt.zero_grad()
        (loss,) = m(q[0].cuda(), q[1].cuda(), a[0].cuda(), a[1].cuda(), b[0].cuda(), b[1].cuda())
        loss.backward()
        opt.step()
        ours.append(float(loss))
    sd_cur = {k: v.detach().clone() for k, v in sd.items()}
    theirs = []
    for i in range(20):
        l, gr = _masked_oracle_loss(sd_cur, [q, a, b], step_seeds[i], nll)
        theirs.append(l)
        sd_cur = {k: (v.cuda() - lr * gr[k]).detach() for k, v in sd_cur.items()}
    print("FirstP dropout losses ours  ", np.round(ours, 4).tolist())
    print("FirstP dropout losses oracle", np.round(theirs, 4).tolist())
    diff = max(abs(x - y) for x, y in zip(ours, theirs))
    assert diff <= 0.02, diff
