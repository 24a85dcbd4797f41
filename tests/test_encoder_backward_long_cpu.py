"""The attention backward of 256-512-token sequences without a GPU: its fp64 reference against autograd, its written bound
against an fp32 emulation of the kernel's arithmetic (tests/encoder_grad_long_refs.py), the new C entry points' argument
checks, and the Python training surface of FirstP, MaxP and the DPR BiEncoder."""
import ctypes as C
import re
from pathlib import Path

import pytest
import torch

from ance_b200 import _lib
from ance_b200.models import BiEncoder, RobertaDot_CLF_ANN_NLL_MultiChunk, RobertaDot_NLL_LN
from ance_b200.synthetic import roberta_base_config
from tests import encoder_grad_long_refs as R
from tests import encoder_grad_refs as G

ROOT = Path(__file__).resolve().parent.parent


def test_reference_matches_fp64_autograd():
    B, L, heads = 2, 256, 2
    qkv, kb, _, dfull = R.inputs(B, L, heads, "fp16", ["holed", "prefix"], 1, 0)
    x = qkv.to(torch.float64).requires_grad_(True)
    q, k, v = G._split(x, B, L, heads)
    s = q @ k.transpose(-1, -2) / 8.0 + kb.to(torch.float64).reshape(B, 1, 1, L) / R.LOG2E
    ctx = G._merge(torch.softmax(s, -1) @ v, B, L, heads)
    (ctx * dfull.to(torch.float64)).sum().backward()
    ref = R.attention_bwd_long_ref(qkv, kb, dfull, B, L, heads)
    assert torch.allclose(ref, x.grad, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
@pytest.mark.parametrize("L", [256, 512])
@pytest.mark.parametrize("cls_only", [0, 1])
def test_bound_covers_the_emulation(fmt, L, cls_only):
    B, heads = 4, 2
    qkv, kb, _, dfull = R.inputs(B, L, heads, fmt, ["full", "prefix", "holed", "allpad"], L + cls_only, cls_only,
                                 late_max=True)
    ref = R.attention_bwd_long_ref(qkv, kb, dfull, B, L, heads)
    tol = R.attention_bwd_long_tol(qkv, kb, dfull, B, L, heads, fmt)
    emu = R.emulate(qkv, kb, dfull, B, L, heads, fmt)
    drop = R.emulate(qkv, kb, dfull, B, L, heads, fmt, drop_rowsum=True)
    err = float(((emu.double() - ref).abs() / tol).max())
    err_drop = float(((drop.double() - ref).abs() / tol).max())
    print(f"{fmt} L{L} cls{cls_only}: emulation err / bound {err:.3f}, rowsum dropped {err_drop:.1f}")
    assert err <= 1.0
    assert err_drop > 1.0
    # the late-maximum rows of sequence 0, head 0 really peak in the last key block
    q, k, _ = G._split(qkv.double(), B, L, heads)
    assert bool((((q[0, 0] @ k[0, 0].T).argmax(-1)) >= L - 64).all())


def test_abi_argument_checks():
    lib = _lib.load()
    p = C.c_void_p(16)
    # a bad format, L outside {256, 384, 512}: refused before any device work
    assert lib.ance_dbg_attention_backward_long(7, p, p, p, 0, 2, 256, 2, p, None) == 1
    for L in (128, 200, 640, 64):
        assert lib.ance_dbg_attention_backward_long(0, p, p, p, 0, 2, L, 2, p, None) == 1
        assert b"L in {256, 384, 512}" in lib.ance_last_error()
    assert lib.ance_dbg_attention_backward_long(0, p, p, p, 0, 2, 512, 17, p, None) == 1
    hdr = (ROOT / "include" / "ance_b200.h").read_text()
    assert '"train_max_len"' in hdr
    assert re.search(r"int ance_dbg_attention_backward_long\(", hdr)


def _cpu_roberta(cls=RobertaDot_NLL_LN):
    return cls(roberta_base_config(num_hidden_layers=1, vocab_size=100))


def test_python_training_surface():
    m = _cpu_roberta()
    with pytest.raises(ValueError, match="max_len"):
        m.set_trainable(True, max_len=300)
    assert m.set_trainable(True, max_len=512) is m and m._train_max_len == 512
    assert m.set_trainable(True)._train_max_len == 128
    bi = BiEncoder(type("A", (), {"num_hidden_layers": 1, "vocab_size": 100})())
    with pytest.raises(NotImplementedError, match="max_len=256"):
        bi.set_trainable(True)
    assert bi.set_trainable(True, max_len=256) is bi and bi._grad_path()
    with pytest.raises(ValueError):
        bi.set_trainable(True, max_len=200)
    bi.set_trainable(False)
    assert not bi._grad_path()
    # MaxP: its 512-token chunks need max_len >= 512; the refusal comes before any device work
    mc = _cpu_roberta(RobertaDot_CLF_ANN_NLL_MultiChunk).set_trainable(True, max_len=256)
    ids = torch.ones(2, 1024, dtype=torch.int64)
    with pytest.raises(_lib.AnceError, match="no backward"):
        mc.body_emb(ids, ids)
    with pytest.raises(_lib.AnceError, match="no backward"):
        mc.encode_lens_multi_chunk_packed(ids.int(), torch.full((2,), 1024, dtype=torch.int32))
