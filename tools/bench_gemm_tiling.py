"""Time the GEMM tilings of ance_dbg_gemm at the four encoder linear-layer shapes, one encoder pass of the flagship
workload (M = 75,776 rows: bench.py's marco_psg step is 64 encoder passes of 592 passages x 128 tokens), 16-bit
operands, each shape with the epilogue its layer uses:
  qkv   N 2304, K 768    bias
  out   N  768, K 768    bias + residual
  ffn1  N 3072, K 768    bias + GELU (logistic form, act 2)
  ffn2  N  768, K 3072   bias + residual
The variants alternate within one process: --rounds rounds, each timing every (shape, variant) over --iters back-to-back
launches between CUDA events after --warmup launches of each.  Prints one JSON line per (shape, variant) with the median
ms and TFLOP/s over the rounds and every round's ms, then one line with the card's name, its power limit and the median
SM clock sampled while the rounds ran.

    python tools/bench_gemm_tiling.py [--variants 0 2] [--shapes qkv out ffn1 ffn2] [--M 75776] [--fmt fp16|bf16]
                                      [--rounds 5] [--iters 50] [--warmup 3]

Variant 0 is the tiling every encoder linear layer runs (BN 128, 4 stages, no cluster); variant 2 the same tile on 2-CTA
clusters that share each B tile through TMA multicast (the search's coarse pass); variant 5 the 128 x 256 tile on two
MMA warpgroups with the epilogue from registers (the encoder's QKV, out-proj and FFN-down).  DESIGN.md §4.3 has the results.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from ance_b200 import _lib  # noqa: E402
from tools.bench_train import ClockSampler, _smi  # noqa: E402

SHAPES = {"qkv": (2304, 768, False, 0), "out": (768, 768, True, 0), "ffn1": (3072, 768, False, 2),
          "ffn2": (768, 3072, True, 0)}   # name -> (N, K, residual, act); every layer has a bias
VARIANT_NAMES = {0: "BN128 4st CG1", 1: "BN128 3st CG1", 2: "BN128 4st CG2", 3: "BN64 6st CG2", 4: "BN64 6st CG1",
                 5: "BN256 3st 2 MMA WG"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", type=int, nargs="+", default=[0, 2])
    ap.add_argument("--shapes", nargs="+", default=list(SHAPES))
    ap.add_argument("--M", type=int, default=75776)
    ap.add_argument("--fmt", choices=["fp16", "bf16"], default="fp16")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    lib = _lib.load()
    dt = torch.float16 if a.fmt == "fp16" else torch.bfloat16
    fmt = _lib.ANCE_FMT_FP16 if a.fmt == "fp16" else _lib.ANCE_FMT_BF16
    st = _lib.current_stream()
    g = torch.Generator(device="cuda").manual_seed(0)
    M = a.M
    ops = {}
    for name in a.shapes:
        N, K, res, act = SHAPES[name]
        A = torch.randn(M, K, generator=g, device="cuda").to(dt)
        W = (torch.randn(N, K, generator=g, device="cuda") * 0.04).to(dt)
        bias = torch.randn(N, generator=g, device="cuda")
        R = torch.randn(M, N, generator=g, device="cuda").to(torch.bfloat16) if res else None
        Cout = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        ops[name] = (N, K, act, A, W, bias, R, Cout)

    def launch(name, v):
        N, K, act, A, W, bias, R, Cout = ops[name]
        rc = lib.ance_dbg_gemm(A.data_ptr(), W.data_ptr(), M, N, K, fmt, v, bias.data_ptr(),
                               None if R is None else R.data_ptr(), act, Cout.data_ptr(), None, st)
        if rc != 0:
            raise RuntimeError(lib.ance_last_error().decode())

    for name in a.shapes:
        for v in a.variants:
            for _ in range(a.warmup):
                launch(name, v)
    torch.cuda.synchronize()
    times = {(n, v): [] for n in a.shapes for v in a.variants}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler() as clk:
        for r in range(a.rounds):
            for name in a.shapes:
                vs = a.variants if r % 2 == 0 else a.variants[::-1]
                for v in vs:
                    e0.record()
                    for _ in range(a.iters):
                        launch(name, v)
                    e1.record()
                    e1.synchronize()
                    times[(name, v)].append(e0.elapsed_time(e1) / a.iters)
    for name in a.shapes:
        N, K = SHAPES[name][:2]
        for v in a.variants:
            t = times[(name, v)]
            ms = statistics.median(t)
            print(json.dumps({"shape": name, "M": M, "N": N, "K": K, "variant": v, "tiling": VARIANT_NAMES.get(v),
                              "fmt": a.fmt, "ms": round(ms, 4), "tflops": round(2.0 * M * N * K / ms / 1e9, 1),
                              "rounds_ms": [round(x, 4) for x in t]}), flush=True)
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "power_limit_w": _smi("power.limit"),
                      "sm_clock_mhz_median": statistics.median(clk.samples) if clk.samples else None,
                      "sm_clock_samples": len(clk.samples)}), flush=True)


if __name__ == "__main__":
    main()
