"""Encoder backward on the GPU: each backward kernel against its fp64 reference (tests/encoder_grad_refs.py) through the
test hooks, then whole-model gradients against fp32 autograd of oracle/encoder_oracle.py, in fp16 and bf16."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from ance_b200 import _lib
from ance_b200.models import RobertaDot_NLL_LN, _CudaEncoder
from ance_b200.synthetic import random_roberta_state_dict, roberta_base_config
from oracle.encoder_oracle import RobertaDotOracle
from tests import encoder_grad_refs as G

pytestmark = pytest.mark.gpu

FMTS = ["fp16", "bf16"]
FMT_CODE = {"fp16": _lib.ANCE_FMT_FP16, "bf16": _lib.ANCE_FMT_BF16}
DT16 = {"fp16": torch.float16, "bf16": torch.bfloat16}
GUARD = 64
SENT32 = 0x7FC0DEAD
LOG2E = 1.4426950408889634
VOCAB = 600   # small vocabulary: ids repeat inside a batch, so the word-gradient scatter-add sums several tokens per row


@pytest.fixture(scope="module")
def gpu_lib():
    assert torch.cuda.is_available()
    return _lib.load()


def _st():
    return _lib.current_stream()


def _guarded32(n):
    buf = torch.full((n + 2 * GUARD,), SENT32, dtype=torch.int32, device="cuda").view(torch.float32)
    return buf, buf[GUARD:GUARD + n]


def _guards_ok(buf, n):
    raw = buf.view(torch.int32)
    assert bool((raw[:GUARD] == SENT32).all()) and bool((raw[GUARD + n:] == SENT32).all()), "a guard was overwritten"


def _check(name, out, ref, tol, pert):
    err, rep = G.discrimination(out.cpu(), ref.cpu(), tol.cpu(), {k: v.cpu() for k, v in pert.items()})
    print(f"{name}: max err / bound {err:.3f}; perturbed max err / bound {rep}")
    assert err <= 1.0, (name, err)
    for k, v in rep.items():
        assert v > 1.0, (name, k, v)


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
def _kbias(B, L, kind, g):
    keep = torch.ones(B, L, dtype=torch.bool)
    for b in range(B):
        if kind == "prefix":
            keep[b, int(torch.randint(1, L + 1, (1,), generator=g)):] = False
        elif kind == "holed":
            keep[b] = torch.rand(L, generator=g) < 0.6
            keep[b, 0] = True
        elif kind == "allpad" and b % 2 == 0:
            keep[b] = False
    return torch.where(keep, 0.0, -10000.0 * LOG2E).reshape(-1).float()


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("L", [8, 32, 64, 128])
@pytest.mark.parametrize("kind", ["prefix", "holed", "allpad"])
def test_attention_backward_kernel(gpu_lib, fmt, L, kind):
    g = torch.Generator().manual_seed(L * 7 + len(kind))
    B, heads = max(2, 256 // L), 4
    H = heads * 64
    qkv = (torch.randn(B * L, 3 * H, generator=g, dtype=torch.float64) * 1.5).to(DT16[fmt])
    kb = _kbias(B, L, kind, g)
    for cls_only in (0, 1):
        rows = B if cls_only else B * L
        dout = torch.randn(rows, H, generator=g, dtype=torch.float64).to(torch.bfloat16)
        dfull = torch.zeros(B * L, H, dtype=torch.bfloat16)
        if cls_only:
            dfull[::L] = dout
        else:
            dfull = dout
        buf, view = _guarded32(B * L * 3 * H)
        qd, kd, dd = qkv.cuda(), kb.cuda(), dout.cuda()
        rc = gpu_lib.ance_dbg_attention_backward(FMT_CODE[fmt], qd.data_ptr(), kd.data_ptr(), dd.data_ptr(), cls_only, B, L,
                                                 heads, view.data_ptr(), _st())
        assert rc == 0, gpu_lib.ance_last_error()
        torch.cuda.synchronize()
        _guards_ok(buf, B * L * 3 * H)
        out = view.view(B * L, 3 * H)
        ref = G.attention_bwd_ref(qkv, kb, dfull, B, L, heads)
        tol = G.attention_bwd_tol(qkv, kb, dfull, B, L, heads)
        pert = {"no softmax Jacobian rowsum": G.attention_bwd_ref(qkv, kb, dfull, B, L, heads, drop_jacobian=True)}
        _check(f"attn bwd {fmt} L{L} {kind} cls{cls_only}", out, ref, tol, pert)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("H", [256, 768, 1024])
def test_layer_norm_backward_kernel(gpu_lib, fmt, H):
    g = torch.Generator().manual_seed(H)
    for rows, f32 in ((1, False), (7, False), (4097, False), (38400, False), (33, True)):
        if rows == 38400 and H != 768:
            continue
        x = torch.randn(rows, H, generator=g, dtype=torch.float64) * 2 + 0.5
        x = x.float() if f32 else x.to(DT16[fmt])
        gamma = (1 + 0.1 * torch.randn(H, generator=g)).float()
        dy = torch.randn(rows, H, generator=g).float()
        xd, gd, dyd = x.cuda(), gamma.cuda(), dy.cuda()
        buf, dx = _guarded32(rows * H)
        dg, db, ds = (torch.full((H,), float("nan"), device="cuda") for _ in range(3))
        rc = gpu_lib.ance_dbg_layer_norm_backward(FMT_CODE[fmt], xd.data_ptr(), int(f32), H, rows, H, gd.data_ptr(), 1e-5,
                                                  dyd.data_ptr(), dx.data_ptr(), dg.data_ptr(), db.data_ptr(),
                                                  ds.data_ptr(), _st())
        assert rc == 0, gpu_lib.ance_last_error()
        torch.cuda.synchronize()
        _guards_ok(buf, rows * H)
        rdx, rg, rb, rs = G.ln_bwd_ref(x, gamma, 1e-5, dy)
        tdx, tg, tb, ts = G.ln_bwd_tol(x, gamma, 1e-5, dy)
        _, sg, sb, _ = G.ln_bwd_ref(x, gamma, 1e-5, dy, swap_gb=True)
        name = f"ln bwd {fmt} H{H} rows{rows} f32{int(f32)}"
        _check(name + " dx", dx.view(rows, H), rdx, tdx, {})
        _check(name + " dgamma", dg, rg, tg, {"dgamma/dbeta swapped": sg})
        _check(name + " dbeta", db, rb, tb, {"dgamma/dbeta swapped": sb})
        _check(name + " dsum", ds, rs, ts, {})


@pytest.mark.parametrize("fmt", FMTS)
def test_gelu_backward_sweep(gpu_lib, fmt):
    u = torch.linspace(-40, 40, 1 << 20, dtype=torch.float64).to(DT16[fmt])
    gd = torch.ones(u.numel(), device="cuda")
    ud = u.cuda()
    rc = gpu_lib.ance_dbg_gelu_backward(FMT_CODE[fmt], ud.data_ptr(), gd.data_ptr(), u.numel(), _st())
    assert rc == 0, gpu_lib.ance_last_error()
    torch.cuda.synchronize()
    _check(f"gelu bwd {fmt}", gd, G.gelu_bwd_ref(u), G.gelu_bwd_tol(u), {"tanh form": G.gelu_bwd_ref(u, tanh_form=True)})


@pytest.mark.parametrize("shape", [(768, 768), (3072, 768), (768, 3072), (2304, 768)])
def test_dgrad_wgrad_on_the_forward_mainloop(gpu_lib, shape):
    """dX = dY W and dW = dY^T X as the backward launches them: the forward's linear on bf16 W^T, and on token-contiguous
    transposes zero-padded to a multiple of 8 tokens (ragged token counts)."""
    N, K = shape   # W [N, K]
    g = torch.Generator().manual_seed(N + K)
    for M in (1, 77, 2563):
        Mp = (M + 7) // 8 * 8
        W = (torch.randn(N, K, generator=g) * 0.04).to(torch.bfloat16)
        dY = torch.randn(M, N, generator=g).to(torch.bfloat16)
        X = torch.randn(M, K, generator=g).to(torch.bfloat16)
        Wt = W.t().contiguous().cuda()
        dYt = torch.zeros(N, Mp, dtype=torch.bfloat16)
        dYt[:, :M] = dY.t()
        Xt = torch.zeros(K, Mp, dtype=torch.bfloat16)
        Xt[:, :M] = X.t()
        dYd, dYtd, Xtd = dY.cuda(), dYt.cuda(), Xt.cuda()
        buf, dX = _guarded32(M * K)
        assert gpu_lib.ance_dbg_linear(_lib.ANCE_FMT_BF16, dYd.data_ptr(), N, M, Wt.data_ptr(), K, N, None, None, 0, 0,
                                       None, dX.data_ptr(), _st()) == 0, gpu_lib.ance_last_error()
        buf2, dW = _guarded32(N * K)
        assert gpu_lib.ance_dbg_linear(_lib.ANCE_FMT_BF16, dYtd.data_ptr(), Mp, N, Xtd.data_ptr(), K, Mp, None, None, 0, 0,
                                       None, dW.data_ptr(), _st()) == 0, gpu_lib.ance_last_error()
        torch.cuda.synchronize()
        _guards_ok(buf, M * K)
        _guards_ok(buf2, N * K)
        _check(f"dgrad N{N} K{K} M{M}", dX.view(M, K), G.gemm_ref(dY, W), G.gemm_tol(dY, W),
               {"W^T in place of W": G.gemm_ref(dY, W.t())} if N == K else {})
        _check(f"wgrad N{N} K{K} M{M}", dW.view(N, K), G.gemm_ref(dY.t(), X), G.gemm_tol(dY.t(), X),
               {"last token dropped": G.gemm_ref(dY[:-1].t(), X[:-1])} if M > 1 else {})


# ------------------------------------------------------------------------------------------------
# whole model
# ------------------------------------------------------------------------------------------------
def _model(fmt, seed=0, n_layer=2):
    cfg = roberta_base_config(num_hidden_layers=n_layer, vocab_size=VOCAB)
    sd = random_roberta_state_dict(seed=seed, n_layer=n_layer, vocab=VOCAB)
    m = RobertaDot_NLL_LN(cfg)
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    m.encoder_operand = fmt
    return m, sd


def _batch(B, L, seed, holed=False):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(max(1, L // 4), L + 1, (B,), generator=g)
    lens[0] = L
    ids = torch.randint(3, VOCAB, (B, L), generator=g)
    mask = torch.arange(L)[None, :] < lens[:, None]
    if holed:
        mask &= torch.rand(B, L, generator=g) < 0.8
        mask[:, 0] = True
    ids = torch.where(torch.arange(L)[None, :] < lens[:, None], ids, torch.full_like(ids, 1))
    ids[:, 0] = 0
    return ids, mask.to(torch.int64)


def _oracle_loss(sd, batches, triplet):
    """fp32 autograd through the oracle on the GPU (TF32 off); returns (loss or sum of weighted embeddings, grads)."""
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        orc = RobertaDotOracle(sd, n_layer=2, device="cuda")
        leaves = {k: v.detach().clone().requires_grad_(True) for k, v in orc.enc.sd.items()}
        orc.enc.sd = leaves
        hw, hb, ng, nb = (t.detach().clone().requires_grad_(True) for t in (orc.head_w, orc.head_b, orc.norm_g, orc.norm_b))

        def emb(ids, mask):
            x = orc.enc._hidden_states(ids.cuda(), mask.cuda())[-1][:, 0]
            return Fn.layer_norm(Fn.linear(x, hw, hb), (768,), ng, nb, 1e-5)

        out = triplet(*[emb(i, m) for i, m in batches])
        out.backward()
        grads = {k: v.grad for k, v in leaves.items()}
        grads.update({"embeddingHead.weight": hw.grad, "embeddingHead.bias": hb.grad, "norm.weight": ng.grad,
                      "norm.bias": nb.grad})
        # nn.Embedding(padding_idx=1) for words and positions (the reference's RobertaEmbeddings): no gradient there
        grads["roberta.embeddings.word_embeddings.weight"][1] = 0
        grads["roberta.embeddings.position_embeddings.weight"][1] = 0
        return float(out.detach()), grads
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


# Per-tensor gate on ||g - g_ref|| / ||g_ref||.  Error model: the backward rounds each GEMM operand to bf16 (u = 2^-9); a
# gradient of the 2-layer model passes through at most ~12 such products from the loss, with independent rounding errors
# adding in quadrature, so ~sqrt(2 * 12) u = 1e-2 relative, plus the forward's stored activations (fp16: 2^-12, bf16:
# 2^-9, through the same depth).  The gate allows 3x that: 0.03 (fp16 forward) / 0.05 (bf16 forward).
GATE = {"fp16": 0.03, "bf16": 0.05}


def _compare_grads(model, grads_ref, fmt, name, extra=0.0):
    """Every parameter's gradient within GATE of the oracle's, relative to the oracle's norm.  The key biases are the
    exception: softmax is invariant to a per-query constant, and q . b_k is one, so their exact gradient is zero and both
    sides hold rounding noise.  They are held to GATE times the norm of the query bias's gradient instead."""
    sdv = model.state_dict(keep_vars=True)
    bad, rels = [], {}
    for k, p in sdv.items():
        ref = grads_ref[k]
        if k.endswith("attention.self.key.bias"):
            scale = grads_ref[k.replace(".key.", ".query.")].norm()
            rel = float(p.grad.norm() / scale)
        else:
            rel = float((p.grad - ref).norm() / ref.norm().clamp_min(1e-30))
        rels[k] = rel
        if not rel <= GATE[fmt] + extra:
            bad.append((k, rel))
    worst = max(rels, key=rels.get)
    print(f"{name} {fmt}: worst per-tensor relative error {rels[worst]:.4f} ({worst}; gate {GATE[fmt] + extra:.4f})")
    assert not bad, f"{name} {fmt}: {bad}"


@pytest.mark.parametrize("fmt", FMTS)
def test_forward_train_equals_forward(gpu_lib, fmt):
    m, _ = _model(fmt)
    enc = m._encoder(torch.device("cuda"))
    for L, holed in ((64, False), (128, True), (8, False)):
        ids, mask = _batch(6, L, L, holed)
        i32, m8 = ids.to(torch.int32).cuda(), mask.to(torch.uint8).cuda()
        ref = enc.forward(i32, None, m8)
        out, ws = enc.forward_train(i32, None, m8)
        assert torch.equal(out, ref)
        lens = mask.sum(1).to(torch.int32).cuda()
        if not holed:
            out2, _ = enc.forward_train(i32, lens, None)
            assert torch.equal(out2, enc.forward(i32, lens, None))


@pytest.mark.parametrize("fmt", FMTS)
def test_parameter_gradients_match_the_oracle(gpu_lib, fmt):
    m, sd = _model(fmt)
    m.set_trainable(True)
    q = _batch(4, 32, 1)
    p = _batch(4, 128, 2, holed=True)
    w = torch.randn(4, 768, generator=torch.Generator().manual_seed(5)).cuda()

    def objective(eq, ep):
        return (eq * w).sum() + (ep * w.flip(0)).sum()

    out = objective(m.query_emb(q[0].cuda(), q[1].cuda()), m.body_emb(p[0].cuda(), p[1].cuda()))
    out.backward()
    _, gref = _oracle_loss(sd, [q, p], objective)
    _compare_grads(m, gref, fmt, "sum(w o emb)")


@pytest.mark.parametrize("fmt", FMTS)
def test_triplet_loss_backward(gpu_lib, fmt):
    m, sd = _model(fmt)
    m.set_trainable(True)
    q, a, b = _batch(4, 64, 3), _batch(4, 128, 4), _batch(4, 128, 5)
    (loss,) = m(q[0].cuda(), q[1].cuda(), a[0].cuda(), a[1].cuda(), b[0].cuda(), b[1].cuda())
    assert loss.grad_fn is not None
    loss.backward()

    def nll(eq, ea, eb):
        lm = torch.stack([(eq * ea).sum(-1), (eq * eb).sum(-1)], dim=1)
        return (-torch.log_softmax(lm, dim=1)[:, 0]).mean()

    lref, gref = _oracle_loss(sd, [q, a, b], nll)
    # the forward's embeddings are within ~1e-3 relative of the oracle's (its own gate); the logits are dot products of
    # two embeddings, so the loss moves by up to ~1 % of its value
    assert abs(float(loss) - lref) <= 0.02 * abs(lref), (float(loss), lref)
    # Unlike a fixed upstream gradient, dL/d(embeddings) here is computed from each side's own embeddings, so it carries
    # the forward's error; every parameter gradient is linear in it and inherits that relative error on top of the
    # backward's own (GATE).  Measure it and widen the gate by twice that.
    orc = RobertaDotOracle(sd, n_layer=2, device="cuda")
    with torch.no_grad():
        ours_e = [m.query_emb(q[0].cuda(), q[1].cuda()), m.body_emb(a[0].cuda(), a[1].cuda()),
                  m.body_emb(b[0].cuda(), b[1].cuda())]
    ref_e = [orc.query_emb(i.cuda(), k.cuda()) for i, k in (q, a, b)]
    up = []
    for es in (ours_e, ref_e):
        leaves = [e.detach().clone().requires_grad_(True) for e in es]
        nll(*leaves).backward()
        up.append(torch.cat([x.grad.reshape(-1) for x in leaves]))
    rel_up = float((up[0] - up[1]).norm() / up[1].norm())
    print(f"triplet NLL {fmt}: upstream gradient relative error {rel_up:.4f}")
    _compare_grads(m, gref, fmt, "triplet NLL", extra=2 * rel_up)


@pytest.mark.parametrize("update", ["torch_sgd", "p_data"])
def test_sgd_trajectory_tracks_the_oracle(gpu_lib, update):
    """20 SGD steps on one fixed triplet batch: the losses follow the fp32 oracle's within 0.02 (each step's gradient
    error, 1e-2 relative, moves the weights by lr x that, far below what changes the loss by 0.02 over 20 steps).
    update = "p_data": the step writes through `p.data`, as the reference trainer's Lamb and transformers' AdamW do, which
    leaves `p._version` unchanged; the training forward must still see the new values."""
    m, sd = _model("fp16", seed=3)
    m.set_trainable(True)
    q, a, b = _batch(8, 64, 6), _batch(8, 128, 7), _batch(8, 128, 8)
    opt = torch.optim.SGD(m.parameters(), lr=0.5)
    ours = []
    for _ in range(20):
        opt.zero_grad()
        (loss,) = m(q[0].cuda(), q[1].cuda(), a[0].cuda(), a[1].cuda(), b[0].cuda(), b[1].cuda())
        loss.backward()
        if update == "torch_sgd":
            opt.step()
        else:
            versions = [p._version for p in m.parameters()]
            for p in m.parameters():
                p.data.add_(p.grad, alpha=-0.5)
            assert [p._version for p in m.parameters()] == versions
        ours.append(float(loss))
    ref_model, _ = _model("fp16", seed=3)
    sd_cur = {k: v.detach().clone() for k, v in ref_model.state_dict().items()}
    theirs = []

    def nll(eq, ea, eb):
        lm = torch.stack([(eq * ea).sum(-1), (eq * eb).sum(-1)], dim=1)
        return (-torch.log_softmax(lm, dim=1)[:, 0]).mean()

    for _ in range(20):
        l, gr = _oracle_loss(sd_cur, [q, a, b], nll)
        theirs.append(l)
        sd_cur = {k: (v - 0.5 * gr[k]).detach() for k, v in sd_cur.items()}
    print("losses ours  ", np.round(ours, 4).tolist())
    print("losses oracle", np.round(theirs, 4).tolist())
    assert theirs[-1] < theirs[0] - 0.05, "the fixed batch should be learnable"
    assert max(abs(x - y) for x, y in zip(ours, theirs)) < 0.02


def test_embedding_backward_kernels(gpu_lib):
    """The embedding sum the backward recomputes, and the scatter-add of its gradient into the word / position rows, with
    ids repeated many times inside the batch (RoBERTa positions, padding rows without gradient) and BERT positions."""
    g = torch.Generator().manual_seed(11)
    vocab, max_pos, H = 50, 514, 768
    for roberta, pad_id, L in ((1, 1, 128), (1, 1, 32), (0, 0, 64)):
        B = 6
        ids = torch.randint(3, vocab, (B, L), generator=g)
        lens = torch.randint(1, L + 1, (B,), generator=g)
        ids = torch.where(torch.arange(L)[None, :] < lens[:, None], ids, torch.full_like(ids, pad_id))
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
        want_E = (word[ids.reshape(-1)] + pos[pids]) + typ[0]   # fp32, the forward's association
        assert torch.equal(E.cpu(), want_E)
        rw, rp = G.embedding_grads_ref(ids, dE, vocab, max_pos, pad_id, bool(roberta))
        tw, tp = G.embedding_grads_tol(ids, dE, vocab, max_pos, pad_id, bool(roberta))
        _, sp = G.embedding_grads_ref(ids, dE, vocab, max_pos, pad_id, bool(roberta), pos_shift=1)
        _check(f"embedding bwd word roberta{roberta} L{L}", dw.view(vocab, H), rw, tw, {})
        _check(f"embedding bwd pos roberta{roberta} L{L}", dp.view(max_pos, H), rp, tp, {"position shifted by one": sp})


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_transpose_bf16_kernel(gpu_lib, kind):
    """Token-contiguous bf16 transposes for wgrad: exact bf16 rounding, strided source rows, zero-filled padding columns."""
    g = torch.Generator().manual_seed(kind)
    dt = {0: torch.float16, 1: torch.bfloat16, 2: torch.float32}[kind]
    for R, C, ld in ((1, 768, 768), (77, 3072, 3072), (2563, 2304, 2304), (8, 768, 128 * 768)):
        src = (torch.randn(R * ld, generator=g) * 3).to(dt).cuda()
        view = src.as_strided((R, C), (ld, 1))
        Rp = (R + 7) // 8 * 8
        dst = torch.full((C, Rp), float("nan"), dtype=torch.bfloat16, device="cuda")
        rc = gpu_lib.ance_dbg_transpose_bf16(kind, src.data_ptr(), ld, R, C, dst.data_ptr(), Rp, _st())
        assert rc == 0, gpu_lib.ance_last_error()
        torch.cuda.synchronize()
        want = torch.zeros(C, Rp, dtype=torch.bfloat16, device="cuda")
        want[:, :R] = view.float().t().to(torch.bfloat16)
        assert torch.equal(dst, want), (kind, R, C, ld)


@pytest.mark.parametrize("fmt", FMTS)
def test_in_place_refresh_equals_rebuild(gpu_lib, fmt):
    m, _ = _model(fmt)
    ids, mask = _batch(8, 128, 9)
    dev = ids.cuda().device
    m.query_emb(ids.cuda(), mask.cuda())
    enc0 = m._encoder(dev)
    with torch.no_grad():
        g = torch.Generator(device="cuda").manual_seed(1)
        for p in m.parameters():
            p.add_(torch.randn(p.shape, generator=g, device="cuda") * 1e-3)
    got = m.query_emb(ids.cuda(), mask.cuda())
    assert m._encoder(dev) is enc0, "a parameter update should refresh the handle in place"
    fresh = _CudaEncoder(m.roberta, _lib.ANCE_ARCH_ROBERTA, 12, 1, (m.embeddingHead, m.norm), m.max_tokens, dev, fmt)
    want = fresh.forward(ids.to(torch.int32).cuda(), None, mask.to(torch.uint8).cuda())
    assert torch.equal(got, want)


def test_long_inputs_and_packed_paths_refuse_gradients(gpu_lib):
    m, _ = _model("fp16")
    m.set_trainable(True)
    ids, mask = _batch(2, 256, 10)
    with pytest.raises(_lib.AnceError, match="no backward"):
        m.query_emb(ids.cuda(), mask.cuda())
    lens = mask.sum(1).to(torch.int32).cuda()
    with pytest.raises(_lib.AnceError, match="no backward"):
        m.encode_lens_varlen(ids[:, :128].to(torch.int32).cuda(), lens.clamp(max=128))
    with torch.no_grad():
        assert m.query_emb(ids.cuda(), mask.cuda()).grad_fn is None
    enc = m._encoder(ids.cuda().device)
    # one backward per training forward: the handle forgets the workspace once its backward has run
    short = _batch(2, 64, 12)
    emb = m.query_emb(short[0].cuda(), short[1].cuda())
    emb.sum().backward(retain_graph=True)
    with pytest.raises(_lib.AnceError, match="already run"):
        emb.sum().backward()
    n = C.c_size_t()
    assert enc.lib.ance_encoder_train_workspace(enc.h, 2, 256, C.byref(n)) == _lib.ANCE_ERR_UNSUPPORTED
