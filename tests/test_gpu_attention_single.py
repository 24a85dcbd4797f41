"""The single-block attention kernel (sequences of up to 128 tokens: dense L = 128, packed L < 128, variable-length row
plans) pinned bit for bit.  Every case of tools/attention_digest.py must reproduce the SHA-256 of the CTX bytes recorded
in tests/golden/attention_single_digests.json, which were written by the row-per-thread kernel that the warp-specialised
one replaced.  The fp64 bound tests of test_gpu_encoder_kernels.py let the arithmetic drift inside the error model; these
do not, so any change to the order or rounding of the single-block softmax shows up here."""
import json
import os

import pytest

from tools import attention_digest as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "attention_single_digests.json")
CASES = D.cases()


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_attention_single_digest_cases_match_golden():
    """The golden file covers exactly the cases the tool generates, and the cases span what the digests are for."""
    names = [n for n, _ in CASES]
    assert sorted(names) == sorted(_golden()), "tools/attention_digest.py cases and the golden file disagree"
    specs = [s for _, s in CASES]
    assert {s["fmt"] for s in specs} == {"fp16", "bf16"}
    assert {s["L"] for s in specs if s["kind"] == "dense"} == {8, 16, 32, 64, 128}
    assert {s["align"] for s in specs if s["kind"] == "plan"} == {1, 16}
    assert {s["seqs"] for s in specs if s["kind"] == "dense" and s["L"] == 128} >= {1, 131, 132, 133, 593}
    assert max(s["sigma"] for s in specs) ** 2 >= 6.0   # peaked: score std of at least 6 nats


@pytest.mark.gpu
@pytest.mark.parametrize("name,spec", CASES, ids=[n for n, _ in CASES])
def test_attention_single_digest(name, spec):
    import torch

    from ance_b200 import _lib
    assert torch.cuda.is_available()
    want = _golden()[name]
    qkv_sha, ctx_sha = D.run(_lib.load(), spec)
    assert qkv_sha == want["qkv_sha256"], f"{name}: the generated inputs changed, not the kernel"
    assert ctx_sha == want["ctx_sha256"], f"{name}: attention output differs from the recorded bits"
