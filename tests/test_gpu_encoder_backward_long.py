"""Encoder backward for inputs of 256-512 tokens on the GPU: the key-blocked attention backward against its fp64 bound
(tests/encoder_grad_long_refs.py), the embedding kernels at 512 positions, the training forward, every stage layer by
layer, and whole-model gradients of FirstP, MaxP and the DPR BiEncoder against fp32 autograd of the oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

from ance_b200 import _lib
from ance_b200.models import BiEncoder, RobertaDot_CLF_ANN_NLL_MultiChunk, RobertaDot_NLL_LN, _CudaEncoder, _param_groups
from ance_b200.synthetic import random_roberta_state_dict, roberta_base_config
from oracle.encoder_oracle import EncoderOracle
from tests import encoder_grad_long_refs as R
from tests import encoder_grad_refs as G
from tests import encoder_layer_refs as LR
from tests.test_gpu_encoder_backward import (VOCAB, _batch, _check, _compare_grads, _guarded32, _guards_ok,
                                             _model, _oracle_loss)
from tests.test_gpu_encoder_backward_layers import GATE_12, _autograd_grads, _check_call, _d_out, _Report, _rel
from tests.test_gpu_encoder_backward_layers import _batch as lbatch
from tests.test_gpu_encoder_backward_layers import _roberta as lroberta

pytestmark = pytest.mark.gpu

FMTS = ["fp16", "bf16"]
FMT_CODE = {"fp16": _lib.ANCE_FMT_FP16, "bf16": _lib.ANCE_FMT_BF16}


@pytest.fixture(scope="module")
def gpu_lib():
    assert torch.cuda.is_available()
    return _lib.load()


def _st():
    return _lib.current_stream()


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("L", [256, 384, 512])
@pytest.mark.parametrize("kind", ["prefix", "holed", "allpad"])
def test_attention_backward_long_kernel(gpu_lib, fmt, L, kind):
    """Sequence 0 is unmasked and its head-0 queries peak in the last key block; the others carry the mask kind, every
    other one all-padding for "allpad".  3 heads, guard words around dQKV."""
    B, heads = 4, 3
    H = heads * 64
    kinds = ["full", kind, kind, "allpad" if kind == "allpad" else "prefix"]
    for cls_only in (0, 1):
        qkv, kb, dout, dfull = R.inputs(B, L, heads, fmt, kinds, L * 3 + len(kind) + cls_only, cls_only, late_max=True)
        buf, view = _guarded32(B * L * 3 * H)
        qd, kd, dd = qkv.cuda(), kb.cuda(), dout.cuda()
        rc = gpu_lib.ance_dbg_attention_backward_long(FMT_CODE[fmt], qd.data_ptr(), kd.data_ptr(), dd.data_ptr(), cls_only,
                                                      B, L, heads, view.data_ptr(), _st())
        assert rc == 0, gpu_lib.ance_last_error()
        torch.cuda.synchronize()
        _guards_ok(buf, B * L * 3 * H)
        out = view.view(B * L, 3 * H)
        ref = R.attention_bwd_long_ref(qkv, kb, dfull, B, L, heads)
        tol = R.attention_bwd_long_tol(qkv, kb, dfull, B, L, heads, fmt)
        pert = {"no softmax Jacobian rowsum": R.attention_bwd_long_ref(qkv, kb, dfull, B, L, heads, drop_rowsum=True)}
        _check(f"attn bwd long {fmt} L{L} {kind} cls{cls_only}", out, ref, tol, pert)
        if cls_only:   # query rows past token 0 have no gradient: dQ exactly zero there
            dq = out.view(B, L, 3 * H)[:, 1:, :H]
            assert bool((dq == 0).all())


def test_embedding_backward_512(gpu_lib):
    """embed_sum / scatter at L = 512: RoBERTa positions up to 513 of 514, BERT's up to 511 of 512."""
    g = torch.Generator().manual_seed(21)
    vocab, H = 50, 768
    for roberta, pad_id, max_pos in ((1, 1, 514), (0, 0, 512)):
        B, L = 3, 512
        ids = torch.randint(3, vocab, (B, L), generator=g)
        lens = torch.tensor([L, 300, 129])
        ids = torch.where(torch.arange(L)[None, :] < lens[:, None], ids, torch.full_like(ids, pad_id))
        ids[1, 50:60] = pad_id   # a hole: RoBERTa positions skip it
        word = torch.randn(vocab, H, generator=g) * 0.1
        pos = torch.randn(max_pos, H, generator=g) * 0.1
        typ = torch.randn(2, H, generator=g) * 0.1
        dE = torch.randn(B * L, H, generator=g)
        idd, wd, pd, td, dEd = (t.cuda() for t in (ids.to(torch.int32).contiguous(), word, pos, typ, dE))
        E = torch.empty(B * L, H, device="cuda")
        bw, dw = _guarded32(vocab * H)
        bp, dp = _guarded32(max_pos * H)
        rc = gpu_lib.ance_dbg_embedding_backward(idd.data_ptr(), B, L, H, roberta, pad_id, vocab, max_pos, wd.data_ptr(),
                                                 pd.data_ptr(), td.data_ptr(), dEd.data_ptr(), E.data_ptr(), dw.data_ptr(),
                                                 dp.data_ptr(), _st())
        assert rc == 0, gpu_lib.ance_last_error()
        torch.cuda.synchronize()
        _guards_ok(bw, vocab * H)
        _guards_ok(bp, max_pos * H)
        pids = G.position_ids(ids, pad_id, bool(roberta)).reshape(-1)
        assert int(pids.max()) == max_pos - 1
        assert torch.equal(E.cpu(), (word[ids.reshape(-1)] + pos[pids]) + typ[0])
        rw, rp = G.embedding_grads_ref(ids, dE, vocab, max_pos, pad_id, bool(roberta))
        tw, tp = G.embedding_grads_tol(ids, dE, vocab, max_pos, pad_id, bool(roberta))
        _, sp = G.embedding_grads_ref(ids, dE, vocab, max_pos, pad_id, bool(roberta), pos_shift=1)
        _check(f"embedding bwd word roberta{roberta} L{L}", dw.view(vocab, H), rw, tw, {})
        _check(f"embedding bwd pos roberta{roberta} L{L}", dp.view(max_pos, H), rp, tp, {"position shifted by one": sp})


# ------------------------------------------------------------------------------------------------
# the training forward and the handle's opt-in
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
def test_forward_train_equals_forward_long(gpu_lib, fmt):
    m, _ = _model(fmt)
    enc = m._encoder(torch.device("cuda"))
    enc.set_param("train_max_len", 512)
    for L in (256, 384, 512):
        ids, mask = _batch(3, L, L, holed=L == 384)
        i32, m8 = ids.to(torch.int32).cuda(), mask.to(torch.uint8).cuda()
        ref = enc.forward(i32, None, m8)
        out, ws = enc.forward_train(i32, None, m8)
        assert torch.equal(out, ref), L
        lo = (C.c_size_t * len(_lib.TRAIN_LAYOUT_FIELDS))()
        _lib.check(enc.lib.ance_dbg_train_layout(enc.h, 3, L, lo))
        assert ws.numel() == lo[len(lo) - 1]


def test_refusals(gpu_lib):
    m, _ = _model("fp16")
    m.set_trainable(True, max_len=256)
    ids, mask = _batch(2, 512, 10)
    with pytest.raises(_lib.AnceError, match="no backward"):
        m.query_emb(ids.cuda(), mask.cuda())
    with pytest.raises(_lib.AnceError, match="no backward"):
        m.query_emb(ids[:, :200].cuda(), mask[:, :200].cuda())
    lens = mask.sum(1).clamp(max=256).to(torch.int32).cuda()
    with pytest.raises(_lib.AnceError, match="no backward"):
        m.encode_lens_packed(ids[:, :256].to(torch.int32).cuda(), lens)
    enc = m._encoder(ids.cuda().device)
    n = C.c_size_t()
    assert enc.lib.ance_encoder_set_param(enc.h, b"train_max_len", 200.0) != 0
    enc.set_param("train_max_len", 512)
    assert enc.lib.ance_encoder_train_workspace(enc.h, 2, 640, C.byref(n)) == _lib.ANCE_ERR_UNSUPPORTED
    assert enc.lib.ance_encoder_train_workspace(enc.h, 2, 200, C.byref(n)) != 0
    assert enc.lib.ance_encoder_train_workspace(enc.h, 2, 512, C.byref(n)) == 0
    i32, m8 = ids.to(torch.int32).cuda(), mask.to(torch.uint8).cuda()
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    out = torch.empty(2, 768, device="cuda")
    for L in (640, 200):
        assert enc.lib.ance_encoder_forward_train(enc.h, i32.data_ptr(), None, m8.data_ptr(), 1, L, ws.data_ptr(),
                                                  out.data_ptr(), _st()) != 0
    lo = (C.c_size_t * len(_lib.TRAIN_LAYOUT_FIELDS))()
    assert enc.lib.ance_dbg_train_layout(enc.h, 2, 640, lo) != 0


@pytest.mark.parametrize("fmt", FMTS)
def test_short_path_untouched_by_the_opt_in(gpu_lib, fmt):
    """A backward at L = 128 on a handle with train_max_len 512 is bit-identical to a default handle's, except the
    word / position rows the scatter-add fills in a run-dependent order."""
    m, _ = _model(fmt)
    dev = torch.device("cuda")
    encs = [_CudaEncoder(m.roberta, _lib.ANCE_ARCH_ROBERTA, 12, 1, (m.embeddingHead, m.norm), 8192, dev, fmt)
            for _ in range(2)]
    encs[1].set_param("train_max_len", 512)
    ids, mask = _batch(6, 128, 31, holed=True)
    d_out = torch.randn(6, 768, generator=torch.Generator().manual_seed(2)).cuda()
    res = []
    for enc in encs:
        out, ws = enc.forward_train(ids.to(torch.int32).cuda(), None, mask.to(torch.uint8).cuda())
        embs, layers, hd = _param_groups(m.roberta, (m.embeddingHead, m.norm))
        mk = lambda ts: [torch.full(t.shape, float("nan"), device="cuda") for t in ts]
        grads = (mk(embs), [mk(l) for l in layers], mk(hd))
        enc.backward(d_out, ws, grads)
        torch.cuda.synchronize()
        res.append((out, grads))
    assert torch.equal(res[0][0], res[1][0])
    flat = lambda g: g[0][2:] + [t for l in g[1] for t in l] + g[2]
    for a, b in zip(flat(res[0][1]), flat(res[1][1])):
        assert torch.equal(a, b)
    for a, b in zip(res[0][1][0][:2], res[1][1][0][:2]):
        assert float((a - b).abs().max()) <= 1e-5 * float(a.abs().max())


# ------------------------------------------------------------------------------------------------
# layer by layer
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
def test_layers_long(gpu_lib, fmt, monkeypatch):
    """Every stage of a 2-layer RoBERTa + head at 3 x 256 and 2 x 512 (holed masks, a length-1 sequence) against the
    fp64 mirror of tests/encoder_layer_refs.py; its attention stage, written for the <= 128 kernel, is replaced for this
    test by the key-blocked kernel's (encoder_grad_long_refs.attention_stage, at the handle's operand format)."""
    short = LR.attention_stage

    def stage(qkv, kbias, dout, edout, B, L, heads):
        if L <= 128:
            return short(qkv, kbias, dout, edout, B, L, heads)
        return R.attention_stage(qkv, kbias, dout, edout, B, L, heads, fmt)

    monkeypatch.setattr(LR, "attention_stage", stage)
    _, e = lroberta(fmt, 2, seed=5)
    e.enc.set_param("train_max_len", 512)
    rep = _Report()
    for i, (B, L) in enumerate(((3, 256), (2, 512))):
        ids, mask = lbatch(B, L, 700 + i)
        _check_call(e, ids, mask, _d_out(B, 768, 70 + i), rep, f"2L {fmt} {B}x{L}")
    rep.show(f"long layers {fmt}")


# ------------------------------------------------------------------------------------------------
# whole model against the oracle
# ------------------------------------------------------------------------------------------------
def _nll(eq, ea, eb):
    lm = torch.stack([(eq * ea).sum(-1), (eq * eb).sum(-1)], dim=1)
    return (-torch.log_softmax(lm, dim=1)[:, 0]).mean()


@pytest.mark.parametrize("fmt", FMTS)
def test_firstp_gradients_match_the_oracle(gpu_lib, fmt):
    """FirstP: triplets of a 64-token query and two 512-token documents on a 2-layer RoBERTa."""
    m, sd = _model(fmt)
    m.set_trainable(True, max_len=512)
    q, a, b = _batch(4, 64, 41), _batch(4, 512, 42, holed=True), _batch(4, 512, 43)
    w = torch.randn(3, 4, 768, generator=torch.Generator().manual_seed(44)).cuda()

    def objective(eq, ea, eb):
        return (eq * w[0]).sum() + (ea * w[1]).sum() + (eb * w[2]).sum()

    objective(m.query_emb(q[0].cuda(), q[1].cuda()), m.body_emb(a[0].cuda(), a[1].cuda()),
              m.body_emb(b[0].cuda(), b[1].cuda())).backward()
    _, gref = _oracle_loss(sd, [q, a, b], objective)
    _compare_grads(m, gref, fmt, "FirstP sum(w o emb)")
    m.zero_grad()
    (loss,) = m(q[0].cuda(), q[1].cuda(), a[0].cuda(), a[1].cuda(), b[0].cuda(), b[1].cuda())
    assert loss.grad_fn is not None
    lref, _ = _oracle_loss(sd, [q, a, b], _nll)
    assert abs(float(loss) - lref) <= 0.02 * abs(lref), (float(loss), lref)


def _maxp(x_embs, q_embs, mask):
    B, full = mask.shape
    first = mask.reshape(B, full // 512, 512)[:, :, 0]
    scores = torch.matmul(q_embs.unsqueeze(1), x_embs.transpose(1, 2))[:, 0, :] + ((1 - first) * -9999).float()
    return scores


@pytest.mark.parametrize("fmt", FMTS)
def test_maxp_gradients_match_the_oracle(gpu_lib, fmt):
    """MaxP: 2 documents x 4 chunks of 512, one chunk all padding, the query e2 - e0 (oracle embeddings of chunks 2 and 0
    of document 1), so that chunk 2 outscores chunk 0 by |e2 - e0|^2 and the best chunk is not the first; objective =
    sum of the MaxP logits."""
    _, sd = _model(fmt)
    m = RobertaDot_CLF_ANN_NLL_MultiChunk(roberta_base_config(num_hidden_layers=2, vocab_size=VOCAB))
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    m.encoder_operand = fmt
    m.set_trainable(True, max_len=512)
    g = torch.Generator().manual_seed(51)
    ids = torch.randint(3, VOCAB, (2, 2048), generator=g)
    ids[:, ::512] = 0
    lens = torch.tensor([2048, 1300])          # document 1: chunk 3 all padding, chunk 2 partly
    mask = (torch.arange(2048)[None, :] < lens[:, None]).to(torch.int64)
    ids = torch.where(mask.bool(), ids, torch.ones_like(ids))
    with torch.no_grad():
        ref_chunks = [_oracle_chunk(sd, ids, mask)]
    qv = (ref_chunks[0][1, 2] - ref_chunks[0][1, 0]).cuda()
    emb = m.body_emb(ids.cuda(), mask.cuda())
    assert emb.shape == (2, 4, 768) and emb.grad_fn is not None
    scores = _maxp(emb, qv.expand(2, 768), mask.cuda())
    assert int(scores[1].argmax()) != 0 and float(scores[1, 3]) < -9000
    scores.max(-1).values.sum().backward()

    def objective(ex):
        return _maxp(ex.reshape(2, 4, 768), qv.expand(2, 768), mask.cuda()).max(-1).values.sum()

    _, gref = _oracle_loss(sd, [(ids.reshape(8, 512), mask.reshape(8, 512))], objective)
    _compare_grads(m, gref, fmt, "MaxP sum of logits")


def _oracle_chunk(sd, ids, mask):
    from oracle.encoder_oracle import RobertaDotOracle
    return RobertaDotOracle(sd, n_layer=2, device="cuda").body_emb_multi_chunk(ids.cuda(), mask.cuda()).cpu()


def _bert_sd(n_layer):
    return {**random_roberta_state_dict(seed=61, n_layer=n_layer, vocab=VOCAB, max_pos=512, head=False,
                                        prefix="question_model."),
            **random_roberta_state_dict(seed=62, n_layer=n_layer, vocab=VOCAB, max_pos=512, head=False,
                                        prefix="ctx_model.")}


@pytest.mark.parametrize("fmt", FMTS)
def test_biencoder_gradients_match_the_oracle(gpu_lib, fmt):
    """DPR at 256 tokens, both forward() forms: (q, a) with in-batch negatives and (loss,) for triplets."""
    sd = _bert_sd(2)
    m = BiEncoder(type("A", (), {"num_hidden_layers": 2, "vocab_size": VOCAB})())
    m.load_state_dict(sd)
    m = m.cuda()
    m.encoder_operand = fmt
    m.set_trainable(True, max_len=256)

    def bert_batch(B, seed):
        ids, mask = _batch(B, 256, seed, holed=False)
        ids = torch.where(mask.bool(), ids, torch.zeros_like(ids))
        ids[:, 0] = 101
        return ids, mask

    q, a, b = bert_batch(6, 71), bert_batch(6, 72), bert_batch(6, 73)
    # Both losses alone leave the ctx encoder's last-LayerNorm bias with an exactly zero gradient (it shifts every passage
    # embedding alike, and each query's softmax weights sum to one), so that tensor, and the ones close to it, would hold
    # rounding noise on both sides.  Fixed-weight terms give every tensor a gradient to compare.
    w = torch.randn(3, 6, 768, generator=torch.Generator().manual_seed(74)).cuda() * 0.05

    def in_batch(eq, ea):
        return -torch.log_softmax(eq @ ea.T, dim=1).diagonal().mean() + (eq * w[0]).sum() + (ea * w[1]).sum()

    def triplet(eq, ea, eb):
        return _nll(eq, ea, eb) + (eq * w[0]).sum() + (ea * w[1]).sum() + (eb * w[2]).sum()

    for form in ("in_batch", "triplet"):
        m.zero_grad()
        if form == "in_batch":
            qe, ae = m(q[0].cuda(), q[1].cuda(), a[0].cuda(), a[1].cuda())
            assert qe.grad_fn is not None and ae.grad_fn is not None
            loss = in_batch(qe, ae)
        else:
            qe, ae, be = m.query_emb(q[0].cuda(), q[1].cuda()), m.body_emb(a[0].cuda(), a[1].cuda()), \
                m.body_emb(b[0].cuda(), b[1].cuda())
            (nll,) = m(q[0].cuda(), q[1].cuda(), a[0].cuda(), a[1].cuda(), b[0].cuda(), b[1].cuda())
            assert nll.grad_fn is not None
            torch.testing.assert_close(nll, _nll(qe, ae, be), rtol=0, atol=0)
            m.zero_grad()
            loss = nll + (qe * w[0]).sum() + (ae * w[1]).sum() + (be * w[2]).sum()
        loss.backward()
        lref, gref = _bert_oracle(sd, q, a, b, in_batch if form == "in_batch" else triplet, form)
        assert abs(float(loss) - lref) <= 0.02 * abs(lref), (form, float(loss), lref)
        # the upstream gradient d loss / d embeddings is computed from each side's own embeddings (see the rdot_nll
        # triplet test): widen the gate by twice its measured relative error
        with torch.no_grad():
            ours = [m.query_emb(q[0].cuda(), q[1].cuda()), m.body_emb(a[0].cuda(), a[1].cuda()),
                    m.body_emb(b[0].cuda(), b[1].cuda())]
        orc = [EncoderOracle(sd, p, "bert", 2, 12, 0, 1e-12, device="cuda") for p in ("question_model.", "ctx_model.")]
        refs = [orc[0].hidden_states(q[0].cuda(), q[1].cuda())[-1][:, 0],
                orc[1].hidden_states(a[0].cuda(), a[1].cuda())[-1][:, 0],
                orc[1].hidden_states(b[0].cuda(), b[1].cuda())[-1][:, 0]]
        up = []
        for es in (ours, refs):
            leaves = [e.detach().clone().requires_grad_(True) for e in es]
            (in_batch(*leaves[:2]) if form == "in_batch" else triplet(*leaves)).backward()
            up.append(torch.cat([x.grad.reshape(-1) for x in leaves[:2 if form == "in_batch" else 3]]))
        rel_up = float((up[0] - up[1]).norm() / up[1].norm())
        _compare_grads(m, gref, fmt, f"BiEncoder {form}", extra=2 * rel_up)


def _bert_oracle(sd, q, a, b, objective, form):
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        orc = [EncoderOracle(sd, p, "bert", 2, 12, 0, 1e-12, device="cuda") for p in ("question_model.", "ctx_model.")]
        for o in orc:
            o.sd = {k: v.detach().clone().requires_grad_(True) for k, v in o.sd.items()}
        emb = lambda o, x: o._hidden_states(x[0].cuda(), x[1].cuda())[-1][:, 0]
        if form == "in_batch":
            out = objective(emb(orc[0], q), emb(orc[1], a))
        else:
            out = objective(emb(orc[0], q), emb(orc[1], a), emb(orc[1], b))
        out.backward()
        grads = {}
        for o in orc:
            for k, v in o.sd.items():
                grads[k] = v.grad if v.grad is not None else torch.zeros_like(v)
            grads[o.p + "embeddings.word_embeddings.weight"][0] = 0   # nn.Embedding(padding_idx=0): no gradient there
        return float(out.detach()), grads
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize("fmt", FMTS)
def test_firstp_twelve_layers_end_to_end(gpu_lib, fmt):
    """12-layer FirstP (4 queries x 64, 2 x 4 documents x 512) under the 12-layer rule: GATE_12 plus twice the measured
    effect of the forward's 16-bit storage on each tensor."""
    sd = random_roberta_state_dict(seed=0, n_layer=12, vocab=VOCAB)
    m = RobertaDot_NLL_LN(roberta_base_config(num_hidden_layers=12, vocab_size=VOCAB))
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    m.encoder_operand = fmt
    m.set_trainable(True, max_len=512)
    batches = [_batch(4, 64, 81), _batch(4, 512, 82), _batch(4, 512, 83, holed=True)]
    w = torch.randn(3, 4, 768, generator=torch.Generator().manual_seed(84)).cuda()

    def objective(eq, ea, eb):
        return (eq * w[0]).sum() + (ea * w[1]).sum() + (eb * w[2]).sum()

    objective(m.query_emb(batches[0][0].cuda(), batches[0][1].cuda()),
              *[m.body_emb(i.cuda(), k.cuda()) for i, k in batches[1:]]).backward()
    ref = _autograd_grads(sd, batches, objective)
    rnd = _autograd_grads(sd, batches, objective, fmt)
    bad, ratios, raw = [], {}, {}
    for k, p in m.state_dict(keep_vars=True).items():
        gate = GATE_12[fmt] + 2 * _rel(rnd[k], ref[k], k, ref)
        raw[k] = _rel(p.grad, ref[k], k, ref)
        ratios[k] = raw[k] / gate
        if not ratios[k] <= 1.0:
            bad.append((k, raw[k], gate))
    top = sorted(ratios, key=ratios.get, reverse=True)[:3]
    print(f"12 layers FirstP {fmt}: relative error / gate, largest: " +
          ", ".join(f"{k} {ratios[k]:.3f} (relative error {raw[k]:.4f})" for k in top))
    assert not bad, bad


def test_firstp_sgd_trajectory_tracks_the_oracle(gpu_lib):
    """20 SGD steps of FirstP on one fixed batch of 4 triplets (64, 512, 512): within 0.02 of the oracle's losses.  At the
    rdot_nll test's lr of 0.5 this batch is fitted in 4 steps (loss 0 in fp32), after which both trajectories are chaotic;
    lr 0.05 keeps the 20 steps on the smooth part."""
    m, _ = _model("fp16", seed=3)
    m.set_trainable(True, max_len=512)
    q, a, b = _batch(4, 64, 91), _batch(4, 512, 92), _batch(4, 512, 93)
    lr = 0.05
    opt = torch.optim.SGD(m.parameters(), lr=lr)
    ours = []
    for _ in range(20):
        opt.zero_grad()
        (loss,) = m(q[0].cuda(), q[1].cuda(), a[0].cuda(), a[1].cuda(), b[0].cuda(), b[1].cuda())
        loss.backward()
        opt.step()
        ours.append(float(loss))
    ref_model, _ = _model("fp16", seed=3)
    sd_cur = {k: v.detach().clone() for k, v in ref_model.state_dict().items()}
    theirs = []
    for _ in range(20):
        l, gr = _oracle_loss(sd_cur, [q, a, b], _nll)
        theirs.append(l)
        sd_cur = {k: (v - lr * gr[k]).detach() for k, v in sd_cur.items()}
    print("FirstP losses ours  ", np.round(ours, 4).tolist())
    print("FirstP losses oracle", np.round(theirs, 4).tolist())
    assert theirs[-1] < theirs[0] - 0.05, "the fixed batch should be learnable"
    assert max(abs(x - y) for x, y in zip(ours, theirs)) < 0.02
