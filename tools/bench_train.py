"""Time one training step of rdot_nll on one GPU: 8 (query, positive, negative) triplets at lengths (64, 128, 128),
forward + NLL loss + backward, with the sm_90a encoder (set_trainable) against fp32 eager autograd of the oracle
(oracle/encoder_oracle.py, TF32 off) on the same GPU.  Prints one JSON line with the median step times, the card's name,
its power limit and the median SM clock sampled during the timed steps; also the same loss without a graph (the inference
forward) and, with --profile, our step's device time per kernel class from a separate run.

    python tools/bench_train.py [--layers 12] [--steps 20] [--warmup 5] [--fmt fp16|bf16] [--profile]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as Fn  # noqa: E402

from ance_b200 import _lib  # noqa: E402
from ance_b200.models import RobertaDot_NLL_LN  # noqa: E402
from ance_b200.synthetic import random_roberta_state_dict, roberta_base_config  # noqa: E402
from oracle.encoder_oracle import RobertaDotOracle  # noqa: E402


def _smi(query):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return r.stdout.strip()


class ClockSampler:
    """Samples the SM clock (MHz) with nvidia-smi while the timed steps run."""

    def __init__(self):
        self.samples, self._stop = [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.is_set():
            try:
                self.samples.append(float(_smi("clocks.sm")))
            except ValueError:
                pass
            self._stop.wait(0.1)

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join()


def _batch(B, L, seed, vocab):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(L // 2, L + 1, (B,), generator=g)
    ids = torch.randint(3, vocab, (B, L), generator=g)
    mask = torch.arange(L)[None, :] < lens[:, None]
    ids = torch.where(mask, ids, torch.ones_like(ids))
    ids[:, 0] = 0
    return ids.cuda(), mask.long().cuda()


def _nll(q, a, b):
    lm = torch.stack([(q * a).sum(-1), (q * b).sum(-1)], dim=1)
    return (-torch.log_softmax(lm, dim=1)[:, 0]).mean()


def _time(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        step()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times), min(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--fmt", default="fp16", choices=("fp16", "bf16"))
    ap.add_argument("--profile", action="store_true", help="also report our step's device time per kernel class")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train needs a GPU")
    cfg = roberta_base_config(num_hidden_layers=args.layers)
    sd = random_roberta_state_dict(seed=0, n_layer=args.layers)
    model = RobertaDot_NLL_LN(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.cuda()
    model.encoder_operand = args.fmt
    model.set_trainable(True)
    q, a, b = _batch(8, 64, 1, cfg.vocab_size), _batch(8, 128, 2, cfg.vocab_size), _batch(8, 128, 3, cfg.vocab_size)

    def ours():
        model.zero_grad(set_to_none=True)
        (loss,) = model(q[0], q[1], a[0], a[1], b[0], b[1])
        loss.backward()

    def ours_forward():   # the same loss without a graph: the inference forward
        with torch.no_grad():
            model(q[0], q[1], a[0], a[1], b[0], b[1])

    orc = RobertaDotOracle(sd, n_layer=args.layers, device="cuda")
    leaves = {k: v.requires_grad_(True) for k, v in orc.enc.sd.items()}
    head = [t.requires_grad_(True) for t in (orc.head_w, orc.head_b, orc.norm_g, orc.norm_b)]

    def emb(ids, mask):
        x = orc.enc._hidden_states(ids, mask)[-1][:, 0]
        return Fn.layer_norm(Fn.linear(x, head[0], head[1]), (768,), head[2], head[3], 1e-5)

    def oracle():
        for t in list(leaves.values()) + head:
            t.grad = None
        _nll(emb(*q), emb(*a), emb(*b)).backward()

    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with ClockSampler() as clk:
            ours_ms, ours_min = _time(ours, args.steps, args.warmup)
            fwd_ms, _ = _time(ours_forward, args.steps, args.warmup)
            orc_ms, orc_min = _time(oracle, args.steps, args.warmup)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    profile = None
    if args.profile:   # a separate, untimed run: the per-launch events slow the host
        _lib.profile_enable(True)
        _lib.profile_read(reset=True)
        for _ in range(args.steps):
            ours()
        torch.cuda.synchronize()
        profile = {k: (round(ms / args.steps, 3), n // args.steps) for k, (ms, n) in _lib.profile_read().items() if n}
        _lib.profile_enable(False)
    name, power = _smi("name,power.limit").split(", ")
    print(json.dumps({
        "workload": f"rdot_nll train step, 8 triplets at (64, 128, 128), {args.layers} layers, hidden 768",
        "operand_fmt": args.fmt, "step_ms_median": round(ours_ms, 3), "step_ms_min": round(ours_min, 3),
        "forward_only_ms_median": round(fwd_ms, 3), "oracle_fp32_eager_ms_median": round(orc_ms, 3), "oracle_fp32_eager_ms_min": round(orc_min, 3),
        "speedup_vs_oracle": round(orc_ms / ours_ms, 2), "gpu": name, "power_limit_w": float(power),
        "sm_clock_mhz_median": statistics.median(clk.samples) if clk.samples else None,
        "steps": args.steps, "warmup": args.warmup,
        "profile_ms_and_launches_per_step": profile}))


if __name__ == "__main__":
    main()
