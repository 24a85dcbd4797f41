"""The backward references of tests/encoder_grad_refs.py on the CPU: each against torch.autograd in fp64, each bound
against an fp32 emulation of the kernel's arithmetic, each perturbed reference outside its bound; the training ABI's
argument checks and no-GPU errors; the opt-in surface of the models."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as Fn

from ance_b200 import _lib
from tests import encoder_grad_refs as G

F64 = torch.float64
LOG2E = 1.4426950408889634


def _attn_case(B=3, L=32, heads=2, seed=0):
    g = torch.Generator().manual_seed(seed)
    H = heads * 64
    qkv = (torch.randn(B * L, 3 * H, generator=g, dtype=F64) * 1.5).to(torch.float16).to(F64)
    keep = torch.rand(B, L, generator=g) < 0.7
    keep[:, 0] = True
    keep[B - 1] = False   # an all-padding sequence
    kb = torch.where(keep, 0.0, -10000.0 * LOG2E).reshape(-1).to(F64)
    dout = torch.randn(B * L, H, generator=g, dtype=F64).to(torch.bfloat16).to(F64)
    return qkv, kb, dout, B, L, heads


def test_attention_ref_matches_autograd():
    qkv, kb, dout, B, L, heads = _attn_case()
    x = qkv.clone().requires_grad_(True)
    q, k, v = G._split(x, B, L, heads)
    s = q @ k.transpose(-1, -2) / 8 + kb.reshape(B, 1, 1, L) / math.log2(math.e)
    o = G._merge(torch.softmax(s, -1) @ v, B, L, heads)
    (o * dout).sum().backward()
    assert torch.allclose(G.attention_bwd_ref(qkv, kb, dout, B, L, heads), x.grad, rtol=1e-10, atol=1e-12)


def _emulate_attention_fp32(qkv, kb, dout, B, L, heads):
    """The kernel's arithmetic in fp32: log2-domain scores, max-subtracted exp2, dS from rowsum(P o dP), / 8."""
    q, k, v = (t.float() for t in G._split(qkv, B, L, heads))
    do = dout.float().reshape(B, L, heads, 64).transpose(1, 2)
    s = (q @ k.transpose(-1, -2)) * (LOG2E / 8) + kb.float().reshape(B, 1, 1, L)
    e = torch.exp2(s - s.amax(-1, keepdim=True))
    p = e / e.sum(-1, keepdim=True)
    dv = p.transpose(-1, -2) @ do
    dp = do @ v.transpose(-1, -2)
    ds = p * (dp - (p * dp).sum(-1, keepdim=True)) * 0.125
    return torch.cat([G._merge(ds @ k, B, L, heads), G._merge(ds.transpose(-1, -2) @ q, B, L, heads),
                      G._merge(dv, B, L, heads)], dim=1)


@pytest.mark.parametrize("L", [8, 64, 128])
def test_attention_bound_covers_fp32_and_rejects_perturbation(L):
    qkv, kb, dout, B, L, heads = _attn_case(B=2, L=L, seed=L)
    ref = G.attention_bwd_ref(qkv, kb, dout, B, L, heads)
    tol = G.attention_bwd_tol(qkv, kb, dout, B, L, heads)
    err, rep = G.discrimination(_emulate_attention_fp32(qkv, kb, dout, B, L, heads), ref, tol,
                                {"no Jacobian rowsum": G.attention_bwd_ref(qkv, kb, dout, B, L, heads, drop_jacobian=True)})
    assert err <= 1.0 and rep["no Jacobian rowsum"] > 10, (err, rep)


def test_layer_norm_ref_matches_autograd_and_bounds():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(37, 768, generator=g, dtype=F64).to(torch.float16).to(F64) * 3 + 1
    gamma = 1 + 0.1 * torch.randn(768, generator=g, dtype=F64)
    beta = 0.1 * torch.randn(768, generator=g, dtype=F64)
    dy = torch.randn(37, 768, generator=g, dtype=F64)
    xv, gv, bv = (t.clone().requires_grad_(True) for t in (x, gamma, beta))
    (Fn.layer_norm(xv, (768,), gv, bv, 1e-5) * dy).sum().backward()
    dx, dg, db, ds = G.ln_bwd_ref(x, gamma, 1e-5, dy)
    assert torch.allclose(dx, xv.grad, rtol=1e-9, atol=1e-12) and torch.allclose(dg, gv.grad) and torch.allclose(db, bv.grad)
    # fp32 emulation (the kernel's order: mean, squared deviations, rsqrt, two row sums)
    xf, gf, dyf = x.float(), gamma.float(), dy.float()
    mean = xf.sum(-1, keepdim=True) / 768
    rstd = torch.rsqrt(((xf - mean) ** 2).sum(-1, keepdim=True) / 768 + 1e-5)
    xh = (xf - mean) * rstd
    gg = dyf * gf
    dxf = rstd * (gg - gg.sum(-1, keepdim=True) / 768 - xh * (gg * xh).sum(-1, keepdim=True) / 768)
    tdx, tg, tb, ts = G.ln_bwd_tol(x, gamma, 1e-5, dy)
    assert G.discrimination(dxf, dx, tdx, {})[0] <= 1.0
    _, sg, sb, _ = G.ln_bwd_ref(x, gamma, 1e-5, dy, swap_gb=True)
    err, rep = G.discrimination((dyf * xh).sum(0), dg, tg, {"swapped": sg})
    assert err <= 1.0 and rep["swapped"] > 10
    err, rep = G.discrimination(dyf.sum(0), db, tb, {"swapped": sb})
    assert err <= 1.0 and rep["swapped"] > 10


def test_gelu_ref_matches_autograd_and_bounds():
    u = torch.linspace(-40, 40, 20001, dtype=F64)
    uv = u.clone().requires_grad_(True)
    Fn.gelu(uv).sum().backward()
    assert torch.allclose(G.gelu_bwd_ref(u), uv.grad, rtol=1e-12, atol=1e-15)
    uf = u.float()
    emu = 0.5 * torch.erfc(-uf * 0.70710678) + uf * 0.39894228 * torch.exp(-0.5 * uf * uf)
    err, rep = G.discrimination(emu, G.gelu_bwd_ref(u), G.gelu_bwd_tol(u), {"tanh": G.gelu_bwd_ref(u, tanh_form=True)})
    assert err <= 1.0 and rep["tanh"] > 10, (err, rep)


def test_gemm_bound_covers_fp32():
    g = torch.Generator().manual_seed(2)
    A = torch.randn(64, 2563, generator=g).to(torch.bfloat16)
    B = torch.randn(2563, 48, generator=g).to(torch.bfloat16)
    assert G.discrimination(A.float() @ B.float(), G.gemm_ref(A, B), G.gemm_tol(A, B), {})[0] <= 1.0


def test_embedding_ref_matches_autograd_and_rejects_shift():
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(3, 20, (4, 16), generator=g)
    ids[:, 12:] = 1
    ids[:, 0] = 0
    dE = torch.randn(64, 32, generator=g, dtype=F64)
    word = torch.zeros(20, 32, dtype=F64, requires_grad=True)
    pos = torch.zeros(40, 32, dtype=F64, requires_grad=True)
    e = Fn.embedding(ids, word, padding_idx=1) + Fn.embedding(G.position_ids(ids, 1), pos, padding_idx=1)
    (e.reshape(64, 32) * dE).sum().backward()
    dw, dp = G.embedding_grads_ref(ids, dE, 20, 40, 1)
    assert torch.allclose(dw, word.grad) and torch.allclose(dp, pos.grad)
    # fp32 emulation of the kernel's scatter-add (one fp32 addition per token into its row, in token order)
    pos_ids = G.position_ids(ids, 1).reshape(-1)
    emu_w = torch.zeros(20, 32).index_add_(0, ids.reshape(-1), dE.float())
    emu_p = torch.zeros(40, 32).index_add_(0, pos_ids, dE.float())
    emu_w[1] = 0
    emu_p[1] = 0
    tw, tp = G.embedding_grads_tol(ids, dE, 20, 40, 1)
    _, sp = G.embedding_grads_ref(ids, dE, 20, 40, 1, pos_shift=1)
    assert G.discrimination(emu_w, dw, tw, {})[0] <= 1.0
    err, rep = G.discrimination(emu_p, dp, tp, {"shifted": sp})
    assert err <= 1.0 and rep["shifted"] > 10, (err, rep)


# ------------------------------------------------------------------------------------------------
# C ABI and Python surface, no GPU
# ------------------------------------------------------------------------------------------------
def test_training_abi_argument_checks(lib):
    n = C.c_size_t()
    assert lib.ance_encoder_train_workspace(None, 1, 64, C.byref(n)) == 1
    assert b"null" in lib.ance_last_error()
    assert lib.ance_encoder_forward_train(None, None, None, None, 1, 64, None, None, None) == 1
    assert lib.ance_encoder_backward(None, None, None, None, None) == 1
    assert lib.ance_encoder_update_weights(None, None, None) == 1
    assert lib.ance_dbg_attention_backward(7, None, None, None, 0, 1, 64, 1, None, None) == 1
    assert b"format" in lib.ance_last_error()
    assert lib.ance_dbg_attention_backward(0, 1, 1, 1, 0, 1, 256, 1, 1, None) == 1
    assert b"L <= 128" in lib.ance_last_error()
    assert lib.ance_dbg_layer_norm_backward(0, 16, 0, 300, 4, 300, 16, 1e-5, 16, 16, None, None, None, None) == 1
    assert lib.ance_dbg_gelu_backward(0, None, None, 5, None) == 1
    assert lib.ance_dbg_embedding_backward(None, 1, 64, 768, 1, 1, 100, 514, None, None, None, None, None, None, None,
                                           None) == 1
    assert lib.ance_dbg_transpose_bf16(3, 16, 8, 8, 8, 16, 8, None) == 1
    assert b"src_kind" in lib.ance_last_error()


def test_training_hooks_fail_without_gpu(lib):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert lib.ance_dbg_attention_backward(0, 16, 16, 16, 0, 1, 64, 1, 16, None) == 2
    assert lib.ance_dbg_layer_norm_backward(0, 16, 0, 768, 4, 768, 16, 1e-5, 16, 16, None, None, None, None) == 2
    assert lib.ance_dbg_gelu_backward(0, 16, 16, 5, None) == 2


def test_opt_in_surface():
    from ance_b200.models import BiEncoder, RobertaDot_NLL_LN
    from ance_b200.synthetic import roberta_base_config
    m = RobertaDot_NLL_LN(roberta_base_config(num_hidden_layers=1, vocab_size=100))
    assert not m._trainable and not m._grad_path()
    assert m.set_trainable(True) is m and m._grad_path()
    with torch.no_grad():
        assert not m._grad_path()
    with pytest.raises(_lib.AnceError, match="no backward"):
        m.encode_lens_packed(torch.zeros(1, 8, dtype=torch.int32), torch.ones(1, dtype=torch.int32))
    m.set_trainable(False)
    assert not m._grad_path()
    with pytest.raises(NotImplementedError):
        BiEncoder(type("A", (), {"num_hidden_layers": 1, "vocab_size": 100})()).set_trainable(True)


# ------------------------------------------------------------------------------------------------
# the layer-by-layer mirror of backward_impl (tests/encoder_layer_refs.py)
# ------------------------------------------------------------------------------------------------
from tests import encoder_layer_refs as LR  # noqa: E402

_P = "roberta."


def _tiny_model(seed, H=256, F=1024, n_layer=2, vocab=40, max_pos=40):
    from oracle.encoder_oracle import random_roberta_state_dict
    sd = random_roberta_state_dict(seed=seed, n_layer=n_layer, hidden=H, ffn=F, vocab=vocab, max_pos=max_pos, head=False)
    g = torch.Generator().manual_seed(seed)
    sd.update({"embeddingHead.weight": torch.randn(H, H, generator=g) * 0.05, "embeddingHead.bias": torch.randn(H, generator=g) * 0.05,
               "norm.weight": 1 + 0.1 * torch.randn(H, generator=g), "norm.bias": 0.1 * torch.randn(H, generator=g)})
    return {k: v.to(F64) for k, v in sd.items()}


def _layer_weights(sd, l, cast=lambda t: t):
    p = f"{_P}encoder.layer.{l}."
    w = lambda n: sd[p + n]
    return {"wqkv": cast(torch.cat([w("attention.self.query.weight"), w("attention.self.key.weight"),
                                    w("attention.self.value.weight")])),
            "wo": cast(w("attention.output.dense.weight")), "w1": cast(w("intermediate.dense.weight")),
            "w2": cast(w("output.dense.weight")), "ln1_g": w("attention.output.LayerNorm.weight"),
            "ln2_g": w("output.LayerNorm.weight")}


_GRAD_NAMES = {"q_w": "attention.self.query.weight", "q_b": "attention.self.query.bias",
               "k_w": "attention.self.key.weight", "k_b": "attention.self.key.bias",
               "v_w": "attention.self.value.weight", "v_b": "attention.self.value.bias",
               "ao_w": "attention.output.dense.weight", "ao_b": "attention.output.dense.bias",
               "ln1_g": "attention.output.LayerNorm.weight", "ln1_b": "attention.output.LayerNorm.bias",
               "ff1_w": "intermediate.dense.weight", "ff1_b": "intermediate.dense.bias",
               "ff2_w": "output.dense.weight", "ff2_b": "output.dense.bias",
               "ln2_g": "output.LayerNorm.weight", "ln2_b": "output.LayerNorm.bias"}
_EMB_NAMES = {"word_emb": "word_embeddings.weight", "pos_emb": "position_embeddings.weight",
              "type_emb": "token_type_embeddings.weight", "emb_ln_g": "LayerNorm.weight", "emb_ln_b": "LayerNorm.bias"}
_HEAD_NAMES = {"head_w": "embeddingHead.weight", "head_b": "embeddingHead.bias", "head_ln_g": "norm.weight",
               "head_ln_b": "norm.bias"}


def _train_forward(sd, ids, mask, n_layer, heads, eps=1e-5, pad=1):
    """What ance_encoder_forward_train saves, in fp64 from the same parameters: per layer x_in, qkv, ctx (all rows) and
    t1, x1, u, ff, t2 (the CLS rows only in the pruned last layer), the key bias, x_final and head_in; plus the output."""
    B, L = ids.shape
    w = lambda n: sd[_P + n]
    ln = lambda x, g, b, e=eps: Fn.layer_norm(x, (x.shape[-1],), g, b, e)
    pos = G.position_ids(ids, pad)
    x = (w("embeddings.word_embeddings.weight")[ids] + w("embeddings.position_embeddings.weight")[pos]) + \
        w("embeddings.token_type_embeddings.weight")[0]
    H = x.shape[-1]
    x = ln(x.reshape(B * L, H), w("embeddings.LayerNorm.weight"), w("embeddings.LayerNorm.bias"))
    kb = torch.where(mask.reshape(-1).bool(), 0.0, -10000.0 * LOG2E).to(F64)
    acts = []
    for l in range(n_layer):
        p = f"encoder.layer.{l}."
        lin = lambda t, n: Fn.linear(t, w(p + n + ".weight"), w(p + n + ".bias"))
        qkv = torch.cat([lin(x, "attention.self.query"), lin(x, "attention.self.key"), lin(x, "attention.self.value")], 1)
        _, _, v = G._split(qkv, B, L, heads)
        ctx = G._merge(G.attention_probs(qkv, kb, B, L, heads) @ v, B, L, heads)
        last = l == n_layer - 1
        cr, xr = (ctx[::L], x[::L]) if last else (ctx, x)
        t1 = lin(cr, "attention.output.dense") + xr
        x1 = ln(t1, w(p + "attention.output.LayerNorm.weight"), w(p + "attention.output.LayerNorm.bias"))
        u = lin(x1, "intermediate.dense")
        ff = Fn.gelu(u)
        t2 = lin(ff, "output.dense") + x1
        acts.append(dict(x_in=x, qkv=qkv, ctx=ctx, t1=t1, x1=x1, u=u, ff=ff, t2=t2))
        x = ln(t2, w(p + "output.LayerNorm.weight"), w(p + "output.LayerNorm.bias"))
    head_in = Fn.linear(x, sd["embeddingHead.weight"], sd["embeddingHead.bias"])
    return acts, kb, x, head_in, ln(head_in, sd["norm.weight"], sd["norm.bias"], 1e-5)


def _tiny_batch(seed, B=3, L=16, vocab=40):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, vocab, (B, L), generator=g)
    lens = torch.tensor([L, 1, L - 5])[:B]   # a sequence of length 1 (its CLS token only)
    mask = (torch.arange(L)[None, :] < lens[:, None])
    mask[0] &= torch.rand(L, generator=g) < 0.7   # a holed mask
    mask[:, 0] = True
    ids = torch.where(torch.arange(L)[None, :] < lens[:, None], ids, torch.full_like(ids, 1))
    ids[:, 0] = 0
    return ids, mask


def _mirror_chain(sd, acts, kb, x_final, head_in, d_out, ids, B, L, heads, n_layer, exact, cast=lambda t: t):
    gh, th = LR.head_bwd_ref(d_out, head_in, x_final, cast(sd["embeddingHead.weight"]), sd["norm.weight"], exact=exact)
    grads, dy = {}, gh["x_final"]
    for n, k in _HEAD_NAMES.items():
        grads[k] = gh[n]
    for l in reversed(range(n_layer)):
        gl, _ = LR.layer_bwd_ref(acts[l], kb, _layer_weights(sd, l, cast), dy, B, L, heads, l == n_layer - 1, 1e-5,
                                 exact=exact)
        for n, k in _GRAD_NAMES.items():
            grads[f"{_P}encoder.layer.{l}.{k}"] = gl[n]
        dy = gl["x_in"]
    w = lambda n: sd[_P + "embeddings." + n]
    ge, _ = LR.embedding_stage_ref(ids, dy, w("word_embeddings.weight"), w("position_embeddings.weight"),
                                   w("token_type_embeddings.weight"), w("LayerNorm.weight"), 1e-5, 1, True)
    for n, k in _EMB_NAMES.items():
        grads[f"{_P}embeddings.{k}"] = ge[n]
    return grads


def test_layer_mirror_at_exact_arithmetic_matches_autograd():
    """The mirror chained head -> pruned last layer -> full layer -> embeddings, with no rounding emulated, equals fp64
    autograd through the oracle's encoder for every parameter."""
    from oracle.encoder_oracle import EncoderOracle
    n_layer, heads = 2, 4
    sd = _tiny_model(0)
    ids, mask = _tiny_batch(0)
    B, L = ids.shape
    leaves = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    acts, kb, x_final, head_in, out = _train_forward(leaves, ids, mask, n_layer, heads)
    orc = EncoderOracle(sd, _P, "roberta", n_layer, heads, 1, 1e-5)
    orc.sd = {k: v for k, v in sd.items() if k.startswith(_P)}
    assert torch.allclose(x_final, orc._hidden_states(ids, mask)[-1][:, 0], rtol=0, atol=1e-12)
    d_out = torch.randn(B, 256, generator=torch.Generator().manual_seed(1), dtype=F64)
    (out * d_out).sum().backward()
    det = lambda d: {k: v.detach() for k, v in d.items()}
    grads = _mirror_chain(sd, [det(a) for a in acts], kb, x_final.detach(), head_in.detach(), d_out, ids, B, L, heads,
                          n_layer, exact=True)
    leaves[_P + "embeddings.word_embeddings.weight"].grad[1] = 0     # padding_idx rows (nn.Embedding)
    leaves[_P + "embeddings.position_embeddings.weight"].grad[1] = 0
    assert set(grads) == set(sd)
    for k, v in grads.items():
        ref = leaves[k].grad
        # the key bias's exact gradient is zero (softmax is shift-invariant per query): both sides hold fp64 noise
        scale = leaves[k.replace(".key.", ".query.")].grad if k.endswith("key.bias") else ref
        assert torch.allclose(v, ref, rtol=1e-9, atol=1e-12 * float(scale.abs().max())), k


def _rb(t):
    return t.float().to(torch.bfloat16).float()


def _ln_bwd32(x, gamma, eps, dy):
    x, gamma, dy = x.float(), gamma.float(), dy.float()
    H = x.shape[1]
    mean = x.sum(-1, keepdim=True) / H
    rstd = torch.rsqrt(((x - mean) ** 2).sum(-1, keepdim=True) / H + eps)
    xh = (x - mean) * rstd
    g = dy * gamma
    dx = rstd * (g - g.sum(-1, keepdim=True) / H - xh * (g * xh).sum(-1, keepdim=True) / H)
    return dx, (dy * xh).sum(0), dy.sum(0), dx.sum(0)


def _gelu_d32(u):
    u = u.float()
    return 0.5 * torch.erfc(-u * 0.70710678) + u * 0.39894228 * torch.exp(-0.5 * u * u)


def _emulate_layer32(a, kb, w, dy, B, L, heads, last, eps):
    """backward_impl's chain for one layer in fp32, bf16 rounding at the same points as the kernels."""
    o = {}
    dT, o["ln2_g"], o["ln2_b"], o["ff2_b"] = _ln_bwd32(a["t2"], w["ln2_g"], eps, dy)
    A = _rb(dT)
    o["ff2_w"] = A.t() @ _rb(a["ff"])
    dU = (A @ _rb(w["w2"])) * _gelu_d32(a["u"])
    o["ff1_b"] = dU.sum(0)
    A = _rb(dU)
    o["ff1_w"] = A.t() @ _rb(a["x1"])
    dX1 = A @ _rb(w["w1"]) + dT
    dT1, o["ln1_g"], o["ln1_b"], o["ao_b"] = _ln_bwd32(a["t1"], w["ln1_g"], eps, dX1)
    A = _rb(dT1)
    ctx = a["ctx"].reshape(B, L, -1)[:, 0] if last else a["ctx"]
    o["ao_w"] = A.t() @ _rb(ctx)
    dC = _rb(A @ _rb(w["wo"]))
    H = dC.shape[1]
    dO = torch.zeros(B * L, H)
    if last:
        dO[::L] = dC
    else:
        dO = dC
    dA = _emulate_attention_fp32(a["qkv"], kb, dO, B, L, heads)
    bias = dA.sum(0)
    o["q_b"], o["k_b"], o["v_b"] = bias[:H], bias[H:2 * H], bias[2 * H:]
    A = _rb(dA)
    for i, n in enumerate(("q_w", "k_w", "v_w")):
        o[n] = A[:, i * H:(i + 1) * H].t() @ _rb(a["x_in"])
    dX = A @ _rb(w["wqkv"])
    dX[::L if last else 1] += dT1
    o["x_in"] = dX
    return o


def _stage_check(name, out, g, t, perturbed):
    """Every output within its bound; every perturbed mirror outside it somewhere.  -> worst err / bound."""
    worst = 0.0
    for k in g:
        err, _ = G.discrimination(out[k], g[k], t[k], {})
        assert err <= 1.0, (name, k, err)
        worst = max(worst, err)
    reps = {}
    for pn, gp in perturbed.items():
        reps[pn] = max(G.discrimination(out[k], g[k], t[k], {pn: gp[k]})[1][pn] for k in g)
    print(f"{name}: worst err / bound {worst:.3f}; perturbed {reps}")
    assert all(v > 1.0 for v in reps.values()), (name, reps)
    return worst


@pytest.mark.parametrize("constructed", [False, True])
def test_layer_bounds_cover_fp32_chain_and_reject_orchestration_bugs(constructed):
    """hidden 256, 2 layers, L = 16, B = 3 (odd B, a length-1 sequence, a holed mask), fp16 activations and weights: each
    stage of the mirror, fed the emulation's own upstream gradient, bounds an fp32 emulation of backward_impl; the
    perturbed mirrors are rejected (all six on the constructed weights, see encoder_layer_refs.construct_for_discrimination)."""
    n_layer, heads, eps = 2, 4, 1e-5
    sd = _tiny_model(1)
    if constructed:
        LR.construct_for_discrimination(sd, n_layer, _P)
    ids, mask = _tiny_batch(1)
    B, L = ids.shape
    with torch.no_grad():
        acts, kb, x_final, head_in, _ = _train_forward(sd, ids, mask, n_layer, heads)
    h16 = lambda t: t.to(torch.float16).to(F64)
    acts = [{k: h16(v) for k, v in a.items()} for a in acts]
    x_final, head_in = h16(x_final), head_in.float().to(F64)
    cast = lambda t: h16(t.float())
    d_out = torch.randn(B, 256, generator=torch.Generator().manual_seed(2)).to(F64)
    # head
    hw = cast(sd["embeddingHead.weight"])
    dT, hg, hb, hbias = _ln_bwd32(head_in, sd["norm.weight"], 1e-5, d_out)
    A = _rb(dT)
    out = {"head_ln_g": hg, "head_ln_b": hb, "head_b": hbias, "head_w": A.t() @ _rb(x_final), "x_final": A @ _rb(hw)}
    g, t = LR.head_bwd_ref(d_out, head_in, x_final, hw, sd["norm.weight"])
    flat = torch.cat([x_final.reshape(-1), torch.zeros(B * L * 256)])
    gp, _ = LR.head_bwd_ref(d_out, head_in, x_final, hw, sd["norm.weight"], perturb="head_x_pitch", x_flat=flat, L=L)
    _stage_check("head", out, g, t, {"head_x_pitch": gp})
    dy = out["x_final"]
    for l in reversed(range(n_layer)):
        last = l == n_layer - 1
        w = _layer_weights(sd, l, cast)
        out = _emulate_layer32(acts[l], kb, w, dy, B, L, heads, last, eps)
        g, t = LR.layer_bwd_ref(acts[l], kb, w, dy.to(F64), B, L, heads, last, eps)
        names = ["gelu_at_ff", "no_ffn_residual"] + (["wo_ctx_pitch"] if last else [])
        if constructed:
            names += ["qk_bias_swap"] + (["ln1_residual_rows"] if last else [])
        pert = {n: LR.layer_bwd_ref(acts[l], kb, w, dy.to(F64), B, L, heads, last, eps, perturb=n)[0] for n in names}
        _stage_check(f"layer {l}", out, g, t, pert)
        dy = out["x_in"]
    # embeddings: the LayerNorm on the fp32 sum, the scatter in token order
    e = lambda n: sd[_P + "embeddings." + n].float()
    E = LR.embedding_sum(ids, e("word_embeddings.weight"), e("position_embeddings.weight"),
                         e("token_type_embeddings.weight"), 1, True, 40).reshape(B * L, 256)
    dE, eg, eb, ds = _ln_bwd32(E, e("LayerNorm.weight"), eps, dy)
    pos = G.position_ids(ids, 1).reshape(-1)
    ww = torch.zeros(40, 256).index_add_(0, ids.reshape(-1), dE)
    pw = torch.zeros(40, 256).index_add_(0, pos, dE)
    ww[1] = 0
    pw[1] = 0
    out = {"word_emb": ww, "pos_emb": pw, "type_emb": torch.stack([ds]), "emb_ln_g": eg, "emb_ln_b": eb}
    g, t = LR.embedding_stage_ref(ids, dy.to(F64), e("word_embeddings.weight"), e("position_embeddings.weight"),
                                  e("token_type_embeddings.weight"), e("LayerNorm.weight"), eps, 1, True)
    _stage_check("embeddings", out, g, t, {})


def test_layer_hooks_argument_checks(lib):
    n = (C.c_size_t * 15)()
    assert lib.ance_dbg_train_layout(None, 1, 64, n) == 1
    assert b"null" in lib.ance_last_error()
    assert lib.ance_encoder_debug_grads(None, -1, None, None) == 1
    assert b"null handle" in lib.ance_last_error()
    assert len(_lib.TRAIN_LAYOUT_FIELDS) == 15
