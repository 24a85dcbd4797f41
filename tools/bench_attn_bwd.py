"""Time the encoder's two attention-backward kernels through their test hooks over the same number of tokens: the
shared-memory kernel at L = 128 (ance_dbg_attention_backward) and the key-blocked tensor-core kernels at L = 256 / 384 /
512 (ance_dbg_attention_backward_long), fp16 and bf16, alternating between the configurations round by round.  Reports
the median ms per call (CUDA events), the algorithmic FLOP rate (5 products x 2 L^2 64 = 640 L^2 per sequence-head), the
card's name, its power limit and the median SM clock sampled while timing.  --dropout P adds, for every configuration,
the dropout kernels at attention-probability rate P (ance_dbg_attention_backward_dropout, the launch the backward makes
after a dropout forward), interleaved with the plain ones.  Prints one JSON line.

    python tools/bench_attn_bwd.py [--tokens 8192] [--heads 12] [--iters 20] [--rounds 5] [--dropout 0.1]
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

LOG2E = 1.4426950408889634


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--heads", type=int, default=12)
    ap.add_argument("--iters", type=int, default=20, help="calls per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="timed windows per configuration, interleaved")
    ap.add_argument("--dropout", type=float, default=0.0, help="also time the dropout kernels at this rate")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attn_bwd needs a GPU")
    lib = _lib.load()
    H = args.heads * 64
    g = torch.Generator(device="cuda").manual_seed(0)
    cfgs = []
    for fmt, dt in (("fp16", torch.float16), ("bf16", torch.bfloat16)):
        for L in (128, 256, 384, 512):
            B = args.tokens // L
            qkv = (torch.randn(B * L, 3 * H, generator=g, device="cuda") * 1.5).to(dt)
            lens = torch.randint(L // 2, L + 1, (B,), generator=g, device="cuda")
            kb = torch.where(torch.arange(L, device="cuda")[None, :] < lens[:, None], 0.0, -10000.0 * LOG2E).reshape(-1)
            dout = torch.randn(B * L, H, generator=g, device="cuda").to(torch.bfloat16)
            dqkv = torch.empty(B * L, 3 * H, device="cuda")
            hook = lib.ance_dbg_attention_backward if L <= 128 else lib.ance_dbg_attention_backward_long
            code = _lib.ANCE_FMT_FP16 if fmt == "fp16" else _lib.ANCE_FMT_BF16
            args_c = (code, qkv.data_ptr(), kb.data_ptr(), dout.data_ptr(), 0, B, L, args.heads, dqkv.data_ptr())
            keep = (qkv, kb, dout, dqkv)
            cfgs.append({"fmt": fmt, "L": L, "B": B, "hook": hook, "args": args_c, "keep": keep, "ms": [], "dropout": 0.0})
            if args.dropout > 0:
                args_d = args_c[:-1] + (args.dropout, 0x5EED, 0, dqkv.data_ptr())
                cfgs.append({"fmt": fmt, "L": L, "B": B, "hook": lib.ance_dbg_attention_backward_dropout, "args": args_d,
                             "keep": keep, "ms": [], "dropout": args.dropout})

    def call(c):
        _lib.check(c["hook"](*c["args"], _lib.current_stream()))

    for c in cfgs:   # warm-up: module load, attributes
        for _ in range(3):
            call(c)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler() as clk:
        for _ in range(args.rounds):
            for c in cfgs:
                e0.record()
                for _ in range(args.iters):
                    call(c)
                e1.record()
                e1.synchronize()
                c["ms"].append(e0.elapsed_time(e1) / args.iters)
    name, power = _smi("name,power.limit").split(", ")
    res = []
    for c in cfgs:
        ms = statistics.median(c["ms"])
        flop = 640.0 * c["L"] ** 2 * c["B"] * args.heads
        res.append({"fmt": c["fmt"], "L": c["L"], "B": c["B"], "dropout": c["dropout"], "kernel": "attn_bwd_kernel" if c["L"] <= 128 else "dq_kernel + dkv_kernel",
                    "ms_median": round(ms, 4), "ms_min": round(min(c["ms"]), 4), "ms_max": round(max(c["ms"]), 4),
                    "tflops": round(flop / ms / 1e9, 2)})
    print(json.dumps({"tokens": args.tokens, "heads": args.heads, "iters": args.iters, "rounds": args.rounds,
                      "gpu": name, "power_limit_w": float(power),
                      "sm_clock_mhz_median": statistics.median(clk.samples) if clk.samples else None, "results": res}))


if __name__ == "__main__":
    main()
