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
