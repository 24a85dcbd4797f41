"""Encoder backward layer by layer on the GPU: every gradient element of every layer, the head and the embedding stage
against the fp64 mirror of tests/encoder_layer_refs.py, fed the kernel's own saved activations (ance_dbg_train_layout)
and its own upstream gradients (ance_encoder_debug_grads); determinism; wgrad at long K."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as Fn

from ance_b200 import _lib
from ance_b200.models import RobertaDot_NLL_LN, _backbone, _CudaEncoder, _param_groups
from ance_b200.synthetic import random_roberta_state_dict, roberta_base_config
from tests import encoder_grad_refs as G
from tests import encoder_layer_refs as LR

pytestmark = pytest.mark.gpu

F64 = torch.float64
FMTS = ["fp16", "bf16"]
DT16 = {"fp16": torch.float16, "bf16": torch.bfloat16}
LOG2E = 1.4426950408889634
VOCAB = 600   # small vocabulary: ids repeat inside a batch


@pytest.fixture(scope="module")
def gpu_lib():
    assert torch.cuda.is_available()
    return _lib.load()


class _Enc:
    """A _CudaEncoder with gradient capture on, plus what the mirror needs of its parameters."""

    def __init__(self, backbone, arch, heads, pad, head, fmt, eps=1e-5):
        dev = torch.device("cuda", torch.cuda.current_device())
        self.enc = _CudaEncoder(backbone, arch, heads, pad, head, 8192, dev, fmt)
        _lib.check(self.enc.lib.ance_encoder_debug_grads(self.enc.h, -1, None, None))
        self.groups = _param_groups(backbone, head)
        self.fmt, self.heads, self.pad, self.eps = fmt, heads, pad, eps
        self.roberta = arch == _lib.ANCE_ARCH_ROBERTA
        self.n_layer = len(self.groups[1])
        self.H = self.groups[0][0].shape[1]

    def run(self, ids, mask, d_out):
        """forward_train + backward of one call -> (gradient groups, captured slots, workspace)."""
        out, ws = self.enc.forward_train(ids.to(torch.int32).cuda(), None, mask.to(torch.uint8).cuda())
        embs, layers, hd = self.groups
        mk = lambda ts: [torch.full(t.shape, float("nan"), device="cuda") for t in ts]
        grads = (mk(embs), [mk(l) for l in layers], mk(hd))
        self.enc.backward(d_out, ws, grads)
        slots = []
        for s in range(self.n_layer + 1):
            buf = torch.empty(min(8192, 4096), self.H, device="cuda")
            _lib.check(self.enc.lib.ance_encoder_debug_grads(self.enc.h, s, buf.data_ptr(), _lib.current_stream()))
            slots.append(buf)
        torch.cuda.synchronize()
        return grads, slots, ws

    def layout(self, B, L):
        out = (C.c_size_t * len(_lib.TRAIN_LAYOUT_FIELDS))()
        _lib.check(self.enc.lib.ance_dbg_train_layout(self.enc.h, B, L, out))
        return dict(zip(_lib.TRAIN_LAYOUT_FIELDS, out))


def _w16(t, fmt):
    return t.detach().float().to(DT16[fmt]).to(F64)


class _Report:
    """Worst error / bound per stage, smallest perturbed error / bound per perturbation."""

    # Rejected on every configuration, random weights included.  "qk_bias_swap" is asserted on the constructed weights
    # (encoder_layer_refs.construct_for_discrimination; on random weights a q bias gradient sits inside the k bias
    # gradient's bound, 0.07 .. 0.69).  "ln1_residual_rows" measured 0.35 .. 2.09 of the last layer's d X_in bound on
    # random weights and ~1.0 on the constructed hidden-768 weights; it is asserted on no-head BERT at hidden 256, where
    # it measured 1.73 .. 2.09, and printed elsewhere.
    ASSERTED = ("gelu_at_ff", "no_ffn_residual", "wo_ctx_pitch", "head_x_pitch")
    ALL = ASSERTED + ("qk_bias_swap", "ln1_residual_rows")

    def __init__(self, asserted=ASSERTED):
        self.worst, self.pert, self.asserted = {}, {}, asserted

    def check(self, stage, name, out, g, t, perturbed=()):
        for k in g:
            err, _ = G.discrimination(out[k], g[k], t[k], {})
            assert err <= 1.0, (name, k, err)
            self.worst[stage] = max(self.worst.get(stage, 0.0), err)
        for pn, gp in dict(perturbed).items():
            rep = max(G.discrimination(out[k], g[k], t[k], {pn: gp[k]})[1][pn] for k in g)
            assert rep > 1.0 or pn not in self.asserted, (name, pn, rep)
            self.pert[pn] = min(self.pert.get(pn, math.inf), rep)

    def show(self, name):
        print(f"{name}: worst err / bound {({k: round(v, 3) for k, v in self.worst.items()})}; "
              f"smallest perturbed err / bound {({k: round(v, 2) for k, v in self.pert.items()})}")


def _check_call(e, ids, mask, d_out, rep, name):
    """One forward_train + backward, every stage against the mirror."""
    B, L = ids.shape
    M, H, fmt, NL = B * L, e.H, e.fmt, e.n_layer
    grads, slots, ws = e.run(ids, mask, d_out)
    lo = e.layout(B, L)
    a16 = lambda off, rows, cols: ws[off:off + rows * cols * 2].view(DT16[fmt]).view(rows, cols).to(F64)
    kb = ws[lo["kbias"]:lo["kbias"] + M * 4].view(torch.float32).to(F64)
    embs, layers, hd = e.groups
    gembs, glayers, ghd = grads
    # head, or the has_head = 0 copy of d_out
    x_final = a16(lo["x_final"], B, H)
    if hd:
        head_in = ws[lo["head_in"]:lo["head_in"] + B * H * 4].view(torch.float32).view(B, H).to(F64)
        g, t = LR.head_bwd_ref(d_out, head_in, x_final, _w16(hd[0], fmt), hd[2].detach())
        out = dict(zip(LR.HEAD_GRADS, ghd), x_final=slots[NL][:B])
        flat = torch.cat([x_final.reshape(-1), torch.zeros(B * L * H, dtype=F64, device=x_final.device)])
        gp, _ = LR.head_bwd_ref(d_out, head_in, x_final, _w16(hd[0], fmt), hd[2].detach(), perturb="head_x_pitch",
                                x_flat=flat, L=L)
        rep.check("head", name + " head", out, g, t, {"head_x_pitch": gp} if B > 1 else {})
    else:
        assert torch.equal(slots[NL][:B], d_out)
    # layers, last to first, each from its own captured upstream gradient
    for l in reversed(range(NL)):
        last = l == NL - 1
        Mr = B if last else M
        base = lo["layers"] + l * lo["per_layer"]
        F = layers[l][10].shape[0]
        act = {"x_in": a16(base + lo["x_in"], M, H), "qkv": a16(base + lo["qkv"], M, 3 * H),
               "ctx": a16(base + lo["ctx"], M, H), "t1": a16(base + lo["t1"], Mr, H), "x1": a16(base + lo["x1"], Mr, H),
               "u": a16(base + lo["u"], Mr, F), "ff": a16(base + lo["ff"], Mr, F), "t2": a16(base + lo["t2"], Mr, H)}
        p = layers[l]
        w = {"wqkv": _w16(torch.cat([p[0], p[2], p[4]]), fmt), "wo": _w16(p[6], fmt), "w1": _w16(p[10], fmt),
             "w2": _w16(p[12], fmt), "ln1_g": p[8].detach(), "ln2_g": p[14].detach()}
        dy = slots[l + 1][:Mr]
        g, t = LR.layer_bwd_ref(act, kb, w, dy, B, L, e.heads, last, e.eps)
        out = dict(zip(LR.LAYER_GRADS, glayers[l]), x_in=slots[l][:M])
        names = ["gelu_at_ff", "no_ffn_residual", "qk_bias_swap"]
        names += ["ln1_residual_rows", "wo_ctx_pitch"] if last and B > 1 else []
        pert = {n: LR.layer_bwd_ref(act, kb, w, dy, B, L, e.heads, last, e.eps, perturb=n)[0] for n in names}
        rep.check("layer", f"{name} layer {l}", out, g, t, pert)
    # embeddings
    g, t = LR.embedding_stage_ref(ids.cuda(), slots[0][:M], *[x.detach() for x in embs[:4]], e.eps, e.pad, e.roberta)
    out = dict(zip(("word_emb", "pos_emb", "type_emb", "emb_ln_g", "emb_ln_b"), gembs))
    rep.check("embeddings", name + " embeddings", out, g, t)
    return grads, slots


def _batch(B, L, seed, vocab=VOCAB, holed=True, cls=0, pad=1):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[0] = L
    if B > 2:
        lens[2] = 1   # a sequence of length 1
    mask = torch.arange(L)[None, :] < lens[:, None]
    if holed:
        mask &= torch.rand(B, L, generator=g) < 0.8
        mask[:, 0] = True
    ids = torch.randint(3, vocab, (B, L), generator=g)
    ids = torch.where(torch.arange(L)[None, :] < lens[:, None], ids, torch.full_like(ids, pad))
    ids[:, 0] = cls
    return ids, mask


def _roberta(fmt, n_layer, seed=0, constructed=False):
    cfg = roberta_base_config(num_hidden_layers=n_layer, vocab_size=VOCAB)
    m = RobertaDot_NLL_LN(cfg)
    sd = random_roberta_state_dict(seed=seed, n_layer=n_layer, vocab=VOCAB)
    if constructed:
        LR.construct_for_discrimination(sd, n_layer, "roberta.")
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    return m, _Enc(m.roberta, _lib.ANCE_ARCH_ROBERTA, 12, 1, (m.embeddingHead, m.norm), fmt)


def _d_out(B, H, seed):
    return torch.randn(B, H, generator=torch.Generator().manual_seed(seed)).cuda()


@pytest.mark.parametrize("fmt", FMTS)
def test_layers_12_bench_shape(gpu_lib, fmt):
    """RoBERTa + head at 12 layers, 8 triplets at the bench shape: a query call (8 x 64) and two passage calls (8 x 128)."""
    _, e = _roberta(fmt, 12)
    rep = _Report()
    for i, (B, L) in enumerate(((8, 64), (8, 128), (8, 128))):
        ids, mask = _batch(B, L, 100 + i)
        _check_call(e, ids, mask, _d_out(B, 768, i), rep, f"12L {fmt} {B}x{L}")
    rep.show(f"12 layers bench shape {fmt}")


@pytest.mark.parametrize("fmt", FMTS)
def test_layers_ragged_batches(gpu_lib, fmt):
    """One 4,096-token call (ln_bwd makes more than one grid pass), and B in {1, 3, 9} x L in {8, 16, 128} with holed
    masks and a length-1 sequence (ragged Bp / Mrp padding in the last layer)."""
    _, e = _roberta(fmt, 2, seed=1)
    rep = _Report()
    shapes = [(32, 128)] + [(B, L) for B in (1, 3, 9) for L in (8, 16, 128)]
    for i, (B, L) in enumerate(shapes):
        ids, mask = _batch(B, L, 200 + i)
        _check_call(e, ids, mask, _d_out(B, 768, 50 + i), rep, f"2L {fmt} {B}x{L}")
    rep.show(f"ragged batches {fmt}")


@pytest.mark.parametrize("fmt", FMTS)
def test_layers_constructed_reject_every_perturbation(gpu_lib, fmt):
    """On weights built so that the q / k bias swap shows (construct_for_discrimination), it is rejected together with
    every perturbation asserted on random weights, each in every configuration that has it."""
    _, e = _roberta(fmt, 2, seed=4, constructed=True)
    rep = _Report(_Report.ASSERTED + ("qk_bias_swap",))
    for i, (B, L) in enumerate(((3, 16), (9, 128), (8, 64))):
        ids, mask = _batch(B, L, 500 + i)
        _check_call(e, ids, mask, _d_out(B, 768, 90 + i), rep, f"constructed {fmt} {B}x{L}")
    rep.show(f"constructed {fmt}")
    assert set(rep.pert) == set(_Report.ALL)


def test_capture_hooks_argument_checks(gpu_lib):
    """ance_encoder_debug_grads refuses reads before capture is enabled, before a captured backward, past the last
    slot and into a null buffer; ance_dbg_train_layout refuses B <= 0 and L > 128 and returns the fields in order."""
    m, _ = _roberta("fp16", 1)
    enc = _CudaEncoder(m.roberta, _lib.ANCE_ARCH_ROBERTA, 12, 1, (m.embeddingHead, m.norm), 8192,
                       torch.device("cuda", torch.cuda.current_device()), "fp16")
    lib, h = enc.lib, enc.h
    buf = torch.empty(4096, 768, device="cuda")
    assert lib.ance_encoder_debug_grads(h, 0, buf.data_ptr(), None) == 1
    assert b"not enabled" in lib.ance_last_error()
    assert lib.ance_encoder_debug_grads(h, -1, None, None) == 0
    assert lib.ance_encoder_debug_grads(h, 0, buf.data_ptr(), None) == 1
    assert b"not captured" in lib.ance_last_error()
    ids, mask = _batch(2, 16, 7)
    groups = _param_groups(m.roberta, (m.embeddingHead, m.norm))
    mk = lambda ts: [torch.empty(t.shape, device="cuda") for t in ts]
    out, ws = enc.forward_train(ids.to(torch.int32).cuda(), None, mask.to(torch.uint8).cuda())
    enc.backward(_d_out(2, 768, 1), ws, (mk(groups[0]), [mk(l) for l in groups[1]], mk(groups[2])))
    assert lib.ance_encoder_debug_grads(h, 1, buf.data_ptr(), None) == 0
    assert lib.ance_encoder_debug_grads(h, 2, buf.data_ptr(), None) == 1
    assert b"bad slot" in lib.ance_last_error()
    assert lib.ance_encoder_debug_grads(h, 0, None, None) == 1
    # a backward of more tokens than capture holds leaves the slots unwritten: reads are refused, not stale
    ids, mask = _batch(64, 128, 8)
    out, ws = enc.forward_train(ids.to(torch.int32).cuda(), None, mask.to(torch.uint8).cuda())
    enc.backward(_d_out(64, 768, 2), ws, (mk(groups[0]), [mk(l) for l in groups[1]], mk(groups[2])))
    assert lib.ance_encoder_debug_grads(h, 0, buf.data_ptr(), None) == 1
    assert b"not captured" in lib.ance_last_error()
    n = (C.c_size_t * 15)()
    assert lib.ance_dbg_train_layout(h, 0, 64, n) == 1 and lib.ance_dbg_train_layout(h, 2, 256, n) == 1
    assert lib.ance_dbg_train_layout(h, 2, 64, n) == 0
    lo = dict(zip(_lib.TRAIN_LAYOUT_FIELDS, n))
    tot = C.c_size_t()
    assert lib.ance_encoder_train_workspace(h, 2, 64, C.byref(tot)) == 0 and lo["total"] == tot.value
    assert lo["ids"] < lo["kbias"] < lo["layers"] < lo["x_final"] < lo["head_in"] < lo["total"]
    torch.cuda.synchronize()


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("H", [256, 512, 1024])
def test_layers_bert_no_head(gpu_lib, fmt, H):
    """BERT positions without a head through the C ABI (has_head = 0: d_out copied into the residual stream), hidden
    256 / 512 / 1024 (ln_bwd<NV = 1, 2, 4>), 2 layers."""
    from oracle.encoder_oracle import random_roberta_state_dict as rsd
    sd = rsd(seed=H, n_layer=2, hidden=H, ffn=4 * H, vocab=VOCAB, max_pos=512, head=False)
    bb = _backbone(VOCAB, H, 2, 4 * H, 512, 1, 0, 1e-12)
    bb.load_state_dict({k[len("roberta."):]: v for k, v in sd.items() if k.startswith("roberta.")}, strict=True)
    bb = bb.cuda()
    e = _Enc(bb, _lib.ANCE_ARCH_BERT, H // 64, 0, None, fmt, eps=1e-12)
    rep = _Report(_Report.ASSERTED + (("ln1_residual_rows",) if H == 256 else ()))
    for i, (B, L) in enumerate(((5, 128), (3, 16))):
        ids, mask = _batch(B, L, 300 + i, cls=101 % VOCAB, pad=0)
        _check_call(e, ids, mask, _d_out(B, H, 70 + i), rep, f"bert H{H} {fmt} {B}x{L}")
    rep.show(f"bert no head H{H} {fmt}")


@pytest.mark.parametrize("fmt", FMTS)
def test_backward_is_deterministic(gpu_lib, fmt):
    """The same forward_train + backward twice: every gradient but the scatter-added word / position rows is
    bit-identical, and so is every captured slot; word / position agree within the scatter bound."""
    _, e = _roberta(fmt, 2, seed=2)
    ids, mask = _batch(8, 128, 400, vocab=40)
    d_out = _d_out(8, 768, 9)
    g1, s1, _ = e.run(ids, mask, d_out)
    g2, s2, _ = e.run(ids, mask, d_out)
    flat = lambda g: g[0][2:] + [t for l in g[1] for t in l] + g[2]
    for i, (x, y) in enumerate(zip(flat(g1), flat(g2))):
        assert torch.equal(x, y), i
    for x, y in zip(s1, s2):
        assert torch.equal(x, y)
    # word / position: the same fp32 additions in another order, each run within the scatter bound of the same exact sum
    emb = [x.detach() for x in e.groups[0][:4]]
    _, t = LR.embedding_stage_ref(ids.cuda(), s1[0][:8 * 128], *emb, e.eps, e.pad, e.roberta)
    for i, k in ((0, "word_emb"), (1, "pos_emb")):
        assert bool(((g1[0][i] - g2[0][i]).abs().double() <= 2 * t[k]).all()), k


@pytest.mark.parametrize("K", [8, 16, 75776])
def test_wgrad_long_k_exact(gpu_lib, K):
    """wgrad's launch at K = max_tokens (75,776) and at one partial K block: small-integer bf16 operands make every fp32
    partial sum exact in any order (|sum| < 2^24), so the result must equal the integer product; a dropped or repeated
    K block changes it."""
    g = torch.Generator().manual_seed(K)
    N_out, N_in = 256, 128
    A = torch.randint(-2, 3, (N_out, K), generator=g)
    X = torch.randint(-2, 3, (N_in, K), generator=g)
    want = (A.double() @ X.double().t()).float()
    assert float(want.abs().max()) < 2 ** 24
    Ad, Xd = A.to(torch.bfloat16).cuda(), X.to(torch.bfloat16).cuda()
    out = torch.full((N_out, N_in), float("nan"), device="cuda")
    rc = gpu_lib.ance_dbg_linear(_lib.ANCE_FMT_BF16, Ad.data_ptr(), K, N_out, Xd.data_ptr(), N_in, K, None, None, 0, 0,
                                 None, out.data_ptr(), _lib.current_stream())
    assert rc == 0, gpu_lib.ance_last_error()
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), want)
    # the last (partial) K block moves most outputs, so dropping or repeating it cannot go unnoticed
    tail = A[:, -(K % 64 or 64):].double() @ X[:, -(K % 64 or 64):].double().t()
    assert float((tail != 0).double().mean()) > 0.5


# ------------------------------------------------------------------------------------------------
# 12 layers end to end against fp32 autograd of the oracle
# ------------------------------------------------------------------------------------------------
# Per-tensor gate on ||g - g_ref|| / ||g_ref|| (the key biases, whose exact gradient is zero, against the query bias's
# gradient norm, as in tests/test_gpu_encoder_backward.py).  Two sources of error:
# * the backward's own bf16 operand roundings.  The 2-layer gate (0.03 fp16 / 0.05 bf16) is 3x the quadrature sum of the
#   ~12 roundings a gradient passes through from the loss; a gradient of layer l of an N-layer model passes through ~6
#   per layer above it, a count linear in depth, so the quadrature sum grows as its square root: sqrt(12 / 2) x.
# * the forward's 16-bit stored activations and weights.  A gradient is evaluated at the rounded forward values; how far
#   that moves it depends on the tensor's conditioning, not on the backward (the last layer's key weights, a sum over
#   keys whose softmax gradients cancel, move most).  It is measured per tensor as fp32 autograd of the same forward
#   with every value the encoder stores rounded to operand_fmt, against the plain fp32 oracle, and the gate widens by
#   twice that, as tests/test_gpu_encoder_backward.py widens its triplet gate by twice the measured upstream error.
GATE_12 = {"fp16": 0.03 * math.sqrt(6.0), "bf16": 0.05 * math.sqrt(6.0)}


def _autograd_grads(sd, batches, objective, fmt=None, n_layer=12, heads=12, pad=1, eps=1e-5):
    """fp32 autograd (TF32 off) of objective(embeddings) through the oracle's arithmetic (oracle/encoder_oracle.py).
    fmt: every value the CUDA encoder stores in 16 bits (linear weights, X, Q / K / V, CTX, T1, X1, FF, T2) is rounded to
    it in the forward, with the gradient passed straight through."""
    r = (lambda t: t) if fmt is None else (lambda t: t + (t.to(DT16[fmt]).float() - t).detach())
    leaves = {k: v.detach().float().cuda().requires_grad_(True) for k, v in sd.items()}
    w = lambda n: leaves["roberta." + n]
    ln = lambda x, p, e=eps: Fn.layer_norm(x, (x.shape[-1],), w(p + ".weight"), w(p + ".bias"), e)

    def emb(ids, mask):
        ids, mask = ids.cuda(), mask.cuda()
        B, L = ids.shape
        pos = G.position_ids(ids.cpu(), pad).cuda()
        x = (w("embeddings.word_embeddings.weight")[ids] + w("embeddings.position_embeddings.weight")[pos]) + \
            w("embeddings.token_type_embeddings.weight")[0]
        x = r(ln(x, "embeddings.LayerNorm"))
        ext = (1.0 - mask.float())[:, None, None, :] * -10000.0
        for l in range(n_layer):
            p = f"encoder.layer.{l}."
            lin = lambda t, n: Fn.linear(t, r(w(p + n + ".weight")), w(p + n + ".bias"))
            hd = lambda t: r(t).view(B, L, heads, 64).transpose(1, 2)
            q, k, v = hd(lin(x, "attention.self.query")), hd(lin(x, "attention.self.key")), hd(lin(x, "attention.self.value"))
            a = r((torch.softmax(q @ k.transpose(-1, -2) / 8.0 + ext, dim=-1) @ v).transpose(1, 2).reshape(B, L, -1))
            x1 = r(ln(r(lin(a, "attention.output.dense") + x), p + "attention.output.LayerNorm"))
            ff = r(Fn.gelu(lin(x1, "intermediate.dense")))
            x = r(ln(r(lin(ff, "output.dense") + x1), p + "output.LayerNorm"))
        hin = Fn.linear(x[:, 0], r(leaves["embeddingHead.weight"]), leaves["embeddingHead.bias"])
        return Fn.layer_norm(hin, (hin.shape[-1],), leaves["norm.weight"], leaves["norm.bias"], 1e-5)

    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        objective(*[emb(i, m) for i, m in batches]).backward()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    g = {k: v.grad for k, v in leaves.items()}
    g["roberta.embeddings.word_embeddings.weight"][pad] = 0   # padding_idx rows (nn.Embedding)
    g["roberta.embeddings.position_embeddings.weight"][pad] = 0
    return g


def _rel(a, ref, k, grads_ref):
    if k.endswith("attention.self.key.bias"):
        return float((a - ref).norm() / grads_ref[k.replace(".key.", ".query.")].norm())
    return float((a - ref).norm() / ref.norm().clamp_min(1e-30))


@pytest.mark.parametrize("fmt", FMTS)
def test_twelve_layers_end_to_end(gpu_lib, fmt):
    """Every parameter gradient of the 12-layer model at the bench shape (8 queries x 64, 2 x 8 passages x 128) against
    fp32 autograd of the oracle, under GATE_12 plus the measured effect of the forward's 16-bit storage."""
    from tests.test_gpu_encoder_backward import _batch as obatch
    sd = random_roberta_state_dict(seed=0, n_layer=12, vocab=VOCAB)
    m = RobertaDot_NLL_LN(roberta_base_config(num_hidden_layers=12, vocab_size=VOCAB))
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    m.encoder_operand = fmt
    m.set_trainable(True)
    batches = [obatch(8, 64, 3), obatch(8, 128, 4), obatch(8, 128, 5)]
    w = torch.randn(3, 8, 768, generator=torch.Generator().manual_seed(6)).cuda()

    def objective(eq, ea, eb):
        return (eq * w[0]).sum() + (ea * w[1]).sum() + (eb * w[2]).sum()

    objective(m.query_emb(batches[0][0].cuda(), batches[0][1].cuda()),
              *[m.body_emb(i.cuda(), k.cuda()) for i, k in batches[1:]]).backward()
    ref = _autograd_grads(sd, batches, objective)
    rnd = _autograd_grads(sd, batches, objective, fmt)
    bad, ratios, raw = [], {}, {}
    for k, p in m.state_dict(keep_vars=True).items():
        fwd = _rel(rnd[k], ref[k], k, ref)
        gate = GATE_12[fmt] + 2 * fwd
        raw[k] = _rel(p.grad, ref[k], k, ref)
        ratios[k] = raw[k] / gate
        if not ratios[k] <= 1.0:
            bad.append((k, ratios[k] * gate, gate))
    top = sorted(ratios, key=ratios.get, reverse=True)[:3]
    print(f"12 layers {fmt}: relative error / gate, largest: " +
          ", ".join(f"{k} {ratios[k]:.3f} (relative error {raw[k]:.4f})" for k in top) +
          f"; largest relative error {max(raw.values()):.4f}; base gate {GATE_12[fmt]:.4f}")
    assert not bad, bad
