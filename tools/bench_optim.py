"""Time the Lamb optimizer step on one GPU: the oracle's eager fp32 Lamb (oracle/lamb_oracle.py: the reference's op
sequence, one pass per tensor, host synchronisations included) against ance_b200.optim.Lamb (three kernels per step).

Parameter sets (seeded, std 0.02; gradients std 1e-3), shaped like the trainers' models:
  rdot_nll  RobertaDot_NLL_LN, RoBERTa-base: 201 tensors, 124,647,168 elements
  dpr       the DPR BiEncoder, two BERT-base: 394 tensors, 217,783,296 elements
For each set, after --warmup steps, --rounds rounds of --steps steps of each optimizer, alternating: median, min and max
of the per-step time (host clock around step() + synchronise), and the fused step's device time per step from CUDA
events around --steps back-to-back steps, its achieved bandwidth at 40 bytes per element (reads p, g, m, v and writes m,
v; reads p, m, v and writes p) and its share of the data-sheet 3.35 TB/s.  Then one full rdot_nll training step
(tools/bench_train.py's psg workload, 12 layers: forward + NLL + backward + clip_grad_norm_(1.0) + step) with each
optimizer.  Card name, power limit and the median SM clock are read in the same run.  Prints one JSON line.

    python tools/bench_optim.py [--steps 20] [--warmup 3] [--rounds 3] [--sets rdot_nll,dpr] [--no-train]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from ance_b200.models import BiEncoder, RobertaDot_NLL_LN  # noqa: E402
from ance_b200.optim import Lamb  # noqa: E402
from ance_b200.synthetic import roberta_base_config  # noqa: E402
from oracle.lamb_oracle import EagerLamb  # noqa: E402
from tools.bench_train import ClockSampler, _setup, _smi  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
BYTES_PER_ELEMENT = 40


def param_shapes(name):
    with torch.device("meta"):
        model = (RobertaDot_NLL_LN(roberta_base_config()) if name == "rdot_nll"
                 else BiEncoder(type("A", (), {"num_hidden_layers": 12})()))
        return [p.shape for p in model.parameters()]


def make_set(shapes, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    params = [torch.nn.Parameter(torch.randn(s, generator=g, device="cuda") * 0.02) for s in shapes]
    for p in params:
        p.grad = torch.randn(p.shape, generator=g, device="cuda") * 1e-3
    return params


def groups(params):
    """The two groups of dpr_utils.get_optimizer (weight decay on matrices, none on vectors), the trainers' eps."""
    return [{"params": [p for p in params if p.dim() > 1], "weight_decay": 0.01},
            {"params": [p for p in params if p.dim() <= 1], "weight_decay": 0.0}]


CLOCK_SAMPLES = []   # SM clock (MHz), sampled during the timed windows only


def time_steps(step, n):
    out = []
    with ClockSampler() as clk:
        for _ in range(n):
            t0 = time.perf_counter()
            step()
            torch.cuda.synchronize()
            out.append((time.perf_counter() - t0) * 1e3)
    CLOCK_SAMPLES.extend(clk.samples)
    return out


def device_ms(step, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def summary(xs):
    return {"median": round(statistics.median(xs), 3), "min": round(min(xs), 3), "max": round(max(xs), 3)}


def bench_set(name, args):
    shapes = param_shapes(name)
    n_el = sum(s.numel() for s in shapes)
    opts = {}
    for label, cls, seed in (("eager", EagerLamb, 1), ("fused", Lamb, 1)):
        opts[label] = cls(groups(make_set(shapes, seed)), lr=1e-4, eps=1e-8)
    for opt in opts.values():
        for _ in range(args.warmup):
            opt.step()
    torch.cuda.synchronize()
    times = {k: [] for k in opts}
    for _ in range(args.rounds):
        for k, opt in opts.items():
            times[k] += time_steps(opt.step, args.steps)
    dev = [device_ms(opts["fused"].step, args.steps) for _ in range(args.rounds)]
    dev_ms = statistics.median(dev)
    floor_ms = BYTES_PER_ELEMENT * n_el / HBM_BYTES_PER_S * 1e3
    res = {"tensors": len(shapes), "elements": n_el, "eager_ms": summary(times["eager"]),
           "fused_ms": summary(times["fused"]), "speedup": round(statistics.median(times["eager"]) /
                                                                 statistics.median(times["fused"]), 2),
           "fused_device_ms_per_step": summary(dev), "bandwidth_floor_ms": round(floor_ms, 3),
           "fused_gb_per_s": round(BYTES_PER_ELEMENT * n_el / dev_ms / 1e6, 1),
           "fused_share_of_3_35_tb_s": round(floor_ms / dev_ms, 3)}
    del opts
    torch.cuda.empty_cache()
    return res


def bench_train_step(args):
    ours, _, _, model = _setup("psg", 12, "fp16")
    params = list(model.parameters())
    opts = {"eager": EagerLamb(params, lr=1e-5, eps=1e-8), "fused": Lamb(params, lr=1e-5, eps=1e-8)}

    def step(opt):
        ours()
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        opt.step()

    for opt in opts.values():
        for _ in range(args.warmup):
            step(opt)
    torch.cuda.synchronize()
    times = {k: [] for k in opts}
    for _ in range(args.rounds):
        for k, opt in opts.items():
            times[k] += time_steps(lambda: step(opt), args.steps)
    return {"workload": "rdot_nll train step, 8 triplets at (64, 128, 128), 12 layers, fp16 operands: forward + NLL + "
                        "backward + clip_grad_norm_ + Lamb step",
            "eager_lamb_ms": summary(times["eager"]), "fused_lamb_ms": summary(times["fused"]),
            "saved_ms": round(statistics.median(times["eager"]) - statistics.median(times["fused"]), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sets", default="rdot_nll,dpr")
    ap.add_argument("--no-train", action="store_true", help="skip the full training step")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim needs a GPU")
    out = {}
    for name in args.sets.split(","):
        out[name] = bench_set(name, args)
    if not args.no_train:
        out["train_step"] = bench_train_step(args)
    name, power = _smi("name,power.limit").split(", ")
    out.update({"gpu": name, "power_limit_w": float(power),
                "sm_clock_mhz_median": statistics.median(CLOCK_SAMPLES) if CLOCK_SAMPLES else None,
                "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
