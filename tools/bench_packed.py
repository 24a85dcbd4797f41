"""Padding-free encoding of 129-512-token inputs (ance_encoder_forward_packed) against the padded paths, on one GPU.

One JSON line per workload (seeded inputs, 12-layer base-size encoders with seeded random weights):
  maxp           rdot_nll_multi_chunk documents at the SURVEY.md cfg-4 lengths (lognormal, median 1,100, sigma 0.8, clipped
                 to [20, 2048]) as 4 x 512 chunks:  dense encode_lens_multi_chunk, encode_lens_bucketed on the chunk view,
                 packed exact (align 16) and packed densest (align 1) encode_lens_multi_chunk_packed
  dpr_passages   BiEncoder.body_emb at L = 256 against body_emb_packed (exact, densest)
  dpr_questions  BiEncoder.query_emb at L = 256 against query_emb_packed (exact, densest)
Per path: docs (or sequences) per second from CUDA events (paths alternate, after warm-up), executed and algorithmic
FLOPs, fill (real tokens / computed rows), attention and GEMM milliseconds from ance_profile_read (a separate profiled
call), and max |diff| against the dense path.  The card name, power limit and SM clocks are read in the same run.

    python tools/bench_packed.py [--docs 1024] [--passages 8192] [--questions 8192] [--iters 3] [--out FILE]
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from ance_b200 import _lib  # noqa: E402
from ance_b200.synthetic import random_roberta_state_dict, roberta_base_config  # noqa: E402

H, F, LAYERS = 768, 3072, 12


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:   # the numbers still stand, but without the card they are incomplete
        return {"error": repr(e)}


def plan(lens, L, max_tokens, align):
    """Rows and attention key blocks the packed forward computes for these lengths (its host planner, every chunk)."""
    lib = _lib.load()
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    rows = blocks = 0
    first = 0
    cap = max_tokens // 128
    row0 = np.zeros(len(lens), dtype=np.int32)
    kv = np.zeros(2 * cap, dtype=np.int32)
    while first < len(lens):
        sub = np.ascontiguousarray(lens[first:])
        n, t = C.c_int(), C.c_int()
        _lib.check(lib.ance_dbg_pack_packed(sub.ctypes.data, len(sub), L, max_tokens, align, row0.ctypes.data, None, None,
                                            kv.ctypes.data, C.byref(n), C.byref(t)))
        rows += t.value * 128
        blocks += int(kv[1:2 * t.value:2].sum())
        first += n.value
    return rows, blocks


def gemm_flop(rows, n_seq, head):
    """Executed encoder GEMM FLOPs: every layer's QKV on all rows, the other GEMMs on all rows except in the last layer
    (CLS rows only), plus the head."""
    full = 2 * (4 * H * H + 2 * H * F)
    return (LAYERS - 1) * rows * full + rows * 2 * 3 * H * H + n_seq * 2 * (H * H + 2 * H * F) + (n_seq * 2 * H * 768 if head else 0)


def attn_flop_tiles(tiles_x_blocks):
    return LAYERS * tiles_x_blocks * 128 * 128 * 4 * H


def algo_flop(lens, head):
    lens = np.asarray(lens, dtype=np.float64)
    return gemm_flop(lens.sum(), len(lens), head) + LAYERS * 4 * H * float((lens ** 2).sum())


def time_paths(paths, iters, warmup):
    for fn in paths.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in paths}
    for _ in range(iters):
        for k, fn in paths.items():   # alternate the paths
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    prof = {}
    _lib.profile_enable(True)
    for k, fn in paths.items():
        _lib.profile_read(reset=True)
        fn()
        p = _lib.profile_read(reset=True)
        prof[k] = {"attn_ms": p["attention"][0], "gemm_ms": p["encoder_gemm"][0]}
    _lib.profile_enable(False)
    return {k: float(np.median(v)) for k, v in ms.items()}, prof


def report(name, n_items, unit, paths, outs, executed, algo, real_tokens, rows, ms, prof, info, extra):
    rec = {"workload": name, "gpu": info, **extra, "algorithmic_tflop": algo / 1e12, "paths": {}}
    ref = outs["dense"]
    for k in paths:
        d = (outs[k] - ref).abs()
        rec["paths"][k] = {f"{unit}_per_s": n_items / ms[k] * 1e3, "ms": ms[k], "speedup_vs_dense": ms["dense"] / ms[k],
                           "executed_tflop": executed[k] / 1e12, "fill": real_tokens / rows[k], "rows": rows[k],
                           **prof[k], "max_abs_vs_dense": float(d.max()),
                           "bit_identical_to_dense": bool(torch.equal(outs[k], ref))}
    return rec


def bench_maxp(args, info):
    from ance_b200.models import RobertaDot_CLF_ANN_NLL_MultiChunk
    dev = torch.device("cuda:0")
    m = RobertaDot_CLF_ANN_NLL_MultiChunk(roberta_base_config())
    m.load_state_dict(random_roberta_state_dict(seed=0), strict=True)
    m = m.to(dev).eval()
    rng = np.random.default_rng(4)
    dl = np.clip(np.round(rng.lognormal(np.log(1100), 0.8, size=args.docs)), 20, 2048).astype(np.int32)
    ids = rng.integers(3, 50265, size=(args.docs, 2048)).astype(np.int32)
    ids[np.arange(2048)[None, :] >= dl[:, None]] = 1
    ids[:, 0] = 0
    ids_d, lens_d, lens_h = torch.from_numpy(ids).to(dev), torch.from_numpy(dl).to(dev), torch.from_numpy(dl)
    clen = np.clip(dl[:, None] - 512 * np.arange(4)[None, :], 0, 512).reshape(-1)
    clen_d = torch.from_numpy(clen.astype(np.int32)).to(dev)
    view = ids_d.reshape(-1, 512)
    bucket_out = torch.empty((len(clen), 768), dtype=torch.float32, device=dev)
    paths = {
        "dense": lambda: m.encode_lens_multi_chunk(ids_d, lens_d),
        "bucketed": lambda: m.encode_lens_bucketed(view, clen_d, out=bucket_out).reshape(args.docs, 4, 768),
        "packed_exact": lambda: m.encode_lens_multi_chunk_packed(ids_d, lens_d, lens_host=lens_h, align=16),
        "packed_densest": lambda: m.encode_lens_multi_chunk_packed(ids_d, lens_d, lens_host=lens_h, align=1),
    }
    outs = {k: fn().clone() for k, fn in paths.items()}
    real = torch.from_numpy(clen > 0).to(dev).reshape(args.docs, 4)
    # the bucketed path encodes an all-padding chunk at the shortest bucket, not at 512: compare the real chunks only
    outs = {k: v[real] for k, v in outs.items()}
    ms, prof = time_paths(paths, args.iters, args.warmup)
    mt = m.max_tokens
    nz = clen[clen > 0]
    n_ch = len(clen)
    rows = {"dense": n_ch * 512}
    b_rows = b_blocks = 0
    for Lb in (8, 16, 32, 64, 128, 256, 384, 512):   # encode_lens_bucketed's buckets for L = 512
        lo = {8: 0, 16: 8, 32: 16, 64: 32, 128: 64, 256: 128, 384: 256, 512: 384}[Lb]
        n = int(((np.maximum(clen, 1) > lo) & (np.maximum(clen, 1) <= Lb)).sum())
        b_rows += n * Lb
        b_blocks += (n * Lb // 128) * max(1, Lb // 128) if Lb >= 128 else (n * Lb + 127) // 128
    rows["bucketed"] = b_rows
    ex = {"dense": gemm_flop(rows["dense"], n_ch, True) + attn_flop_tiles(n_ch * 4 * 4),
          "bucketed": gemm_flop(b_rows, n_ch, True) + attn_flop_tiles(b_blocks)}
    for k, a in (("packed_exact", 16), ("packed_densest", 1)):
        r, blk = plan(nz, 512, mt, a)
        rows[k] = r
        ex[k] = gemm_flop(r, len(nz), True) + attn_flop_tiles(blk)
    return report("maxp", args.docs, "docs", paths, outs, ex, algo_flop(nz, True), int(nz.sum()), rows, ms, prof, info,
                  {"docs": args.docs, "lengths": "lognormal(log 1100, 0.8) clipped to [20, 2048], 4 x 512 chunks",
                   "chunks": n_ch, "empty_chunks": int((clen == 0).sum())})


def bench_dpr(args, info, which):
    from ance_b200.models import BiEncoder
    dev = torch.device("cuda:0")
    m = BiEncoder()
    sd = {**random_roberta_state_dict(seed=1, vocab=30522, max_pos=512, head=False, prefix="question_model."),
          **random_roberta_state_dict(seed=2, vocab=30522, max_pos=512, head=False, prefix="ctx_model.")}
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    L = 256
    rng = np.random.default_rng(5 if which == "passages" else 6)
    if which == "passages":
        n, dist = args.passages, "normal(160, 30) rounded, clipped to [20, 256]"
        lens = np.clip(np.round(rng.normal(160, 30, size=n)), 20, L).astype(np.int64)
        dense_fn, packed_fn = m.body_emb, m.body_emb_packed
    else:
        n, dist = args.questions, "uniform integers in [10, 30]"
        lens = rng.integers(10, 31, size=n)
        dense_fn, packed_fn = m.query_emb, m.query_emb_packed
    ids = np.zeros((n, L), dtype=np.int64)
    ids[np.arange(L)[None, :] < lens[:, None]] = rng.integers(1000, 30522, size=int(lens.sum()))
    ids[:, 0] = 101
    ids[np.arange(n), lens - 1] = 102
    ids_h = torch.from_numpy(ids)
    x = ids_h.to(dev)
    mask = x != 0
    paths = {
        "dense": lambda: dense_fn(x, mask),
        "packed_exact": lambda: packed_fn(x, align=16, ids_host=ids_h),
        "packed_densest": lambda: packed_fn(x, align=1, ids_host=ids_h),
    }
    outs = {k: fn().clone() for k, fn in paths.items()}
    ms, prof = time_paths(paths, args.iters, args.warmup)
    rows = {"dense": n * L}
    ex = {"dense": gemm_flop(n * L, n, False) + attn_flop_tiles(n * (L // 128) ** 2)}
    for k, a in (("packed_exact", 16), ("packed_densest", 1)):
        r, blk = plan(lens, L, m.max_tokens, a)
        rows[k] = r
        ex[k] = gemm_flop(r, n, False) + attn_flop_tiles(blk)
    return report("dpr_" + which, n, "seqs", paths, outs, ex, algo_flop(lens, False), int(lens.sum()), rows, ms, prof,
                  info, {"seqs": n, "L": L, "lengths": dist})


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--docs", type=int, default=1024)
    ap.add_argument("--passages", type=int, default=8192)
    ap.add_argument("--questions", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_packed.py measures on a GPU; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    with torch.no_grad():
        recs = [bench_maxp(args, gpu_info()), bench_dpr(args, gpu_info(), "passages"), bench_dpr(args, gpu_info(), "questions")]
    for r in recs:
        line = json.dumps(r)
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
