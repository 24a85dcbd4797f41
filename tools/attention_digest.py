"""SHA-256 digests of the single-block attention output (sequences of up to 128 tokens) on seeded inputs.

    python tools/attention_digest.py --out tests/golden/attention_single_digests.json

runs ance_dbg_attention on every case of cases() (fp16 and bf16; dense L = 128 with all-real, prefix-padded, holed and
all-padding masks; peaked scores; packed L in {8, 16, 32, 64}; variable-length row plans at align 1 and 16; grids
smaller than, equal to and larger than the SM count) and writes, per case, the digest of the CTX bytes and of the QKV
bytes it was given.  tests/test_gpu_attention_single.py recomputes the same cases and compares: the single-block
arithmetic is pinned bit for bit, not only inside the fp64 bounds of test_gpu_encoder_kernels.py.
Inputs come from numpy's PCG64 streams (stable across numpy versions), so the input digests only change if a case does."""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

LOG2E = 1.4426950408889634
HEAD = 64
MAX_TOKENS = 75776          # plan capacity: 592 tiles of 128 rows (the benchmark's passage batch)


def cases():
    """(name, dict) per case.  kinds: 'dense' (L-token sequences back to back, mask kinds cycled per sequence),
    'plan' (variable-length row plan of ance_dbg_pack_packed at L = 128)."""
    out = []
    for fmt in ("fp16", "bf16"):
        for tiles, heads in ((1, 1), (131, 1), (132, 1), (133, 1), (264, 1), (265, 1), (133, 12), (593, 12)):
            out.append((f"{fmt}_dense128_t{tiles}_h{heads}", dict(kind="dense", fmt=fmt, L=128, seqs=tiles, heads=heads,
                                                                  sigma=1.0, seed=tiles * 16 + heads)))
        out.append((f"{fmt}_dense128_peaked", dict(kind="dense", fmt=fmt, L=128, seqs=133, heads=12, sigma=2.5, seed=7)))
        for L in (8, 16, 32, 64):
            seqs = 133 * 128 // L + 3   # a partial last tile
            out.append((f"{fmt}_packed{L}", dict(kind="dense", fmt=fmt, L=L, seqs=seqs, heads=12, sigma=1.0, seed=L)))
            out.append((f"{fmt}_packed{L}_peaked", dict(kind="dense", fmt=fmt, L=L, seqs=seqs, heads=3, sigma=2.5,
                                                        seed=100 + L)))
        for align in (1, 16):
            out.append((f"{fmt}_plan_align{align}", dict(kind="plan", fmt=fmt, seqs=300, heads=12, sigma=1.0,
                                                         seed=200 + align, align=align)))
            out.append((f"{fmt}_plan_align{align}_peaked", dict(kind="plan", fmt=fmt, seqs=300, heads=2, sigma=2.5,
                                                                seed=300 + align, align=align)))
    return out


def _masks(rng, seqs, L):
    """keep [seqs * L]: per sequence, cycling all-real / prefix-padded / holed / all-padding."""
    keep = np.zeros((seqs, L), dtype=bool)
    for b in range(seqs):
        k = b % 4
        if k == 0:
            keep[b] = True
        elif k == 1:
            keep[b, :int(rng.integers(1, L + 1))] = True
        elif k == 2:
            keep[b] = rng.random(L) < 0.7
            keep[b, 0] = True
    return keep.reshape(-1)


def _plan(lib, lens, align):
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    row0 = np.zeros(len(lens), np.int32)
    lo = np.zeros(MAX_TOKENS, np.int32)
    hi = np.zeros(MAX_TOKENS, np.int32)
    placed, tiles = C.c_int(), C.c_int()
    rc = lib.ance_dbg_pack_packed(lens.ctypes.data, len(lens), 128, MAX_TOKENS, align, row0.ctypes.data,
                                  lo.ctypes.data, hi.ctypes.data, None, C.byref(placed), C.byref(tiles))
    assert rc == 0, lib.ance_last_error()
    assert placed.value == len(lens), "plan did not place every sequence"
    n = tiles.value * 128
    return lo[:n], hi[:n], n


def inputs(lib, spec):
    """(n_tokens, L, qkv uint16 [n, 3 H], kbias fp32 [n], row_lo, row_hi) of a case, on the host."""
    rng = np.random.default_rng(spec["seed"])
    heads = spec["heads"]
    lo = hi = None
    if spec["kind"] == "dense":
        L = spec["L"]
        n = spec["seqs"] * L
        keep = _masks(rng, spec["seqs"], L)
        kbias = np.where(keep, 0.0, -10000.0 * LOG2E).astype(np.float32)
    else:
        L = 128
        lens = rng.integers(1, 129, spec["seqs"])
        lens[:6] = (1, 16, 31, 32, 127, 128)
        lo, hi, n = _plan(lib, lens, spec["align"])
        kbias = np.zeros(n, np.float32)
    x = rng.standard_normal((n, 3 * heads * HEAD), dtype=np.float32)
    x[:, :2 * heads * HEAD] *= spec["sigma"]   # Q and K: score std sigma^2 (in nats, after the 1/8 scale)
    import torch
    dt = torch.float16 if spec["fmt"] == "fp16" else torch.bfloat16
    qkv = torch.from_numpy(x).to(dt).view(torch.int16).numpy().view(np.uint16)
    return n, L, qkv, kbias, lo, hi


def run(lib, spec):
    """(sha256 of QKV bytes, sha256 of CTX bytes) of one case."""
    import torch
    from ance_b200 import _lib
    n, L, qkv, kbias, lo, hi = inputs(lib, spec)
    heads = spec["heads"]
    dev = torch.device("cuda")
    qkv_d = torch.from_numpy(qkv.view(np.int16)).to(dev)
    kb_d = torch.from_numpy(kbias).to(dev)
    lo_d = torch.from_numpy(lo).to(dev) if lo is not None else None
    hi_d = torch.from_numpy(hi).to(dev) if hi is not None else None
    ctx = torch.full((n, heads * HEAD), 0x7E5A, dtype=torch.int16, device=dev)
    fmt = _lib.ANCE_FMT_FP16 if spec["fmt"] == "fp16" else _lib.ANCE_FMT_BF16
    rc = lib.ance_dbg_attention(fmt, qkv_d.data_ptr(), n, L, heads, kb_d.data_ptr(),
                                None if lo_d is None else lo_d.data_ptr(), None if hi_d is None else hi_d.data_ptr(),
                                None, ctx.data_ptr(), _lib.current_stream())
    assert rc == 0, lib.ance_last_error()
    torch.cuda.synchronize()
    return hashlib.sha256(qkv.tobytes()).hexdigest(), hashlib.sha256(ctx.cpu().numpy().tobytes()).hexdigest()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    from ance_b200 import _lib
    lib = _lib.load()
    res = {}
    for name, spec in cases():
        qd, cd = run(lib, spec)
        res[name] = {"qkv_sha256": qd, "ctx_sha256": cd}
        print(name, cd[:16], flush=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
