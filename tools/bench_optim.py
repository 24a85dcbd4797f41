"""Time an optimizer step on one GPU.  --optimizer lamb (the default): the oracle's eager fp32 Lamb (oracle/lamb_oracle.py:
the reference's op sequence, one pass per tensor, host synchronisations included) against ance_b200.optim.Lamb (three
kernels per step).  --optimizer adamw: the oracle's eager fp32 AdamW (oracle/adamw_oracle.py: transformers 2.3.0's op
sequence, one pass per tensor) against ance_b200.optim.AdamW (one kernel per step), with torch.optim.AdamW(fused=True)
timed alongside for context only (its arithmetic differs: eps after the bias correction, decay before the update).

Parameter sets (seeded, std 0.02; gradients std 1e-3), shaped like the trainers' models:
  rdot_nll  RobertaDot_NLL_LN, RoBERTa-base: 201 tensors, 124,647,168 elements
  dpr       the DPR BiEncoder, two BERT-base: 394 tensors, 217,783,296 elements
For each set, after --warmup steps, --rounds rounds of --steps steps of each optimizer, alternating: median, min and max
of the per-step time (host clock around step() + synchronise), and the fused step's device time per step from CUDA
events around --steps back-to-back steps, its achieved bandwidth at 40 bytes per element for Lamb (reads p, g, m, v and
writes m, v; reads p, m, v and writes p) or 28 for AdamW (reads p, g, m, v and writes p, m, v) and its share of the
data-sheet 3.35 TB/s (for AdamW from the kernel's own time, the library's `optim` profile class, as the step's
event-timed window also holds the gaps in which the GPU waits for the host).  Then one full training step with each of the eager and the fused optimizer: for Lamb
tools/bench_train.py's psg workload (rdot_nll, 12 layers), for AdamW its dpr workload (the DPR BiEncoder, 16 pairs at
256, in-batch negatives, 12 layers); forward + loss + backward + clip_grad_norm_(1.0) + step.  Card name, power limit
and the median SM clock are read in the same run.  Prints one JSON line.

    python tools/bench_optim.py [--optimizer lamb|adamw] [--steps 20] [--warmup 3] [--rounds 3] [--sets rdot_nll,dpr]
                                [--no-train]
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

from ance_b200 import _lib  # noqa: E402
from ance_b200.models import BiEncoder, RobertaDot_NLL_LN  # noqa: E402
from ance_b200.optim import AdamW, Lamb  # noqa: E402
from ance_b200.synthetic import roberta_base_config  # noqa: E402
from oracle.adamw_oracle import EagerAdamW  # noqa: E402
from oracle.lamb_oracle import EagerLamb  # noqa: E402
from tools.bench_train import ClockSampler, _setup, _smi  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
BYTES_PER_ELEMENT = 40
ADAMW_BYTES_PER_ELEMENT = 28


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


def kernel_ms(step, n):
    """Device time of the library's optimizer kernels alone (the `optim` profile class: CUDA events around each launch),
    per step: unlike device_ms it leaves out the gaps in which the GPU waits for the host to enqueue the next step."""
    _lib.profile_enable(True)
    _lib.profile_read(reset=True)
    for _ in range(n):
        step()
    ms, _ = _lib.profile_read()["optim"]
    _lib.profile_enable(False)
    return ms / n


def _torch_fused_adamw(params, **kw):
    return torch.optim.AdamW(params, fused=True, **kw)


def bench_set_adamw(name, args):
    shapes = param_shapes(name)
    n_el = sum(s.numel() for s in shapes)
    arms = (("eager", EagerAdamW), ("fused", AdamW), ("torch_fused", _torch_fused_adamw))
    opts = {label: cls(groups(make_set(shapes, 1)), lr=1e-4, eps=1e-8) for label, cls in arms}
    for opt in opts.values():
        for _ in range(args.warmup):
            opt.step()
    torch.cuda.synchronize()
    times = {k: [] for k in opts}
    for _ in range(args.rounds):
        for k, opt in opts.items():
            times[k] += time_steps(opt.step, args.steps)
    dev = {k: [device_ms(opts[k].step, args.steps) for _ in range(args.rounds)] for k in ("fused", "torch_fused")}
    kern = [kernel_ms(opts["fused"].step, args.steps) for _ in range(args.rounds)]
    kern_ms = statistics.median(kern)
    floor_ms = ADAMW_BYTES_PER_ELEMENT * n_el / HBM_BYTES_PER_S * 1e3
    res = {"tensors": len(shapes), "elements": n_el, "eager_ms": summary(times["eager"]),
           "fused_ms": summary(times["fused"]), "speedup": round(statistics.median(times["eager"]) /
                                                                 statistics.median(times["fused"]), 2),
           "fused_device_ms_per_step": summary(dev["fused"]), "fused_kernel_ms_per_step": summary(kern),
           "bandwidth_floor_ms": round(floor_ms, 3),
           "fused_kernel_gb_per_s": round(ADAMW_BYTES_PER_ELEMENT * n_el / kern_ms / 1e6, 1),
           "fused_kernel_share_of_3_35_tb_s": round(floor_ms / kern_ms, 3),
           "torch_fused_ms_context_only": summary(times["torch_fused"]),
           "torch_fused_device_ms_per_step_context_only": summary(dev["torch_fused"])}
    del opts
    torch.cuda.empty_cache()
    return res


def bench_train_step_adamw(args):
    ours, _, _, model = _setup("dpr", 12, "fp16")
    params = list(model.parameters())
    opts = {"eager": EagerAdamW(groups(params), lr=1e-5, eps=1e-8), "fused": AdamW(groups(params), lr=1e-5, eps=1e-8)}

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
    return {"workload": "DPR BiEncoder in-batch train step, 16 pairs at 256, 12 layers, fp16 operands: forward + "
                        "in-batch NLL + backward + clip_grad_norm_ + AdamW step",
            "eager_adamw_ms": summary(times["eager"]), "fused_adamw_ms": summary(times["fused"]),
            "saved_ms": round(statistics.median(times["eager"]) - statistics.median(times["fused"]), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--optimizer", default="lamb", choices=("lamb", "adamw"))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sets", default="rdot_nll,dpr")
    ap.add_argument("--no-train", action="store_true", help="skip the full training step")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim needs a GPU")
    adamw = args.optimizer == "adamw"
    out = {"optimizer": "adamw"} if adamw else {}
    for name in args.sets.split(","):
        out[name] = (bench_set_adamw if adamw else bench_set)(name, args)
    if not args.no_train:
        out["train_step"] = (bench_train_step_adamw if adamw else bench_train_step)(args)
    name, power = _smi("name,power.limit").split(", ")
    out.update({"gpu": name, "power_limit_w": float(power),
                "sm_clock_mhz_median": statistics.median(CLOCK_SAMPLES) if CLOCK_SAMPLES else None,
                "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
