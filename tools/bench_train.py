"""Time one training step on one GPU: forward + NLL loss + backward, with the sm_90a encoder (set_trainable) against fp32
eager autograd of the oracle (oracle/encoder_oracle.py, TF32 off) on the same GPU.  Workloads (--workload):
  psg     rdot_nll, 8 (query, positive, negative) triplets at lengths (64, 128, 128) (MS MARCO passages; the default)
  firstp  rdot_nll, 8 triplets at (64, 512, 512) (FirstP documents)
  maxp    rdot_nll_multi_chunk, 2 triplets, queries of 64, documents of 4 chunks x 512 (MaxP)
  dpr     the DPR BiEncoder (two BERTs), 16 (question, passage) pairs at 256 with in-batch negatives  Prints one JSON line with the median step times, the card's name,
its power limit and the median SM clock sampled during the timed steps; also the same loss without a graph (the inference
forward) and, with --profile, our step's device time per kernel class from a separate run.  --dropout instead times our
step with the reference's training-mode dropout (set_trainable(..., dropout=True): 0.1 at every site) and without it,
alternating in --rounds rounds of --steps steps within one process, and prints both medians and every round's median
(with --profile also the device time per kernel class of each, from separate runs).

    python tools/bench_train.py [--workload psg|firstp|maxp|dpr] [--layers 12] [--steps 20] [--warmup 5]
                                [--fmt fp16|bf16] [--profile] [--dropout [--rounds 3]]
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
from ance_b200.models import BiEncoder, RobertaDot_CLF_ANN_NLL_MultiChunk, RobertaDot_NLL_LN  # noqa: E402
from ance_b200.synthetic import random_roberta_state_dict, roberta_base_config  # noqa: E402
from oracle.encoder_oracle import EncoderOracle, RobertaDotOracle  # noqa: E402

WORKLOADS = {
    "psg": "rdot_nll train step, 8 triplets at (64, 128, 128)",
    "firstp": "rdot_nll (FirstP) train step, 8 triplets at (64, 512, 512)",
    "maxp": "rdot_nll_multi_chunk (MaxP) train step, 2 triplets, queries of 64, documents of 4 x 512",
    "dpr": "DPR BiEncoder train step, 16 pairs at 256, in-batch negatives",
}


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


def _batch(B, L, seed, vocab, pad=1, cls=0):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(L // 2, L + 1, (B,), generator=g)
    ids = torch.randint(3, vocab, (B, L), generator=g)
    mask = torch.arange(L)[None, :] < lens[:, None]
    ids = torch.where(mask, ids, torch.full_like(ids, pad))
    ids[:, 0] = cls
    return ids.cuda(), mask.long().cuda()


def _in_batch(q, a):
    return -torch.log_softmax(q @ a.T, dim=1).diagonal().mean()


def _maxp_nll(q, a, b, mask_a, mask_b):
    def logit(x, mask):
        B = x.shape[0]
        first = mask.reshape(B, x.shape[1], -1)[:, :, 0]
        return (torch.matmul(q.unsqueeze(1), x.transpose(1, 2))[:, 0, :] + ((1 - first) * -9999).float()).max(-1).values
    lm = torch.stack([logit(a, mask_a), logit(b, mask_b)], dim=1)
    return (-torch.log_softmax(lm, dim=1)[:, 0]).mean()


def _setup(workload, layers, fmt):
    """-> (ours: one training step, ours_forward: the same loss without a graph, oracle: its fp32 eager step)."""
    if workload == "dpr":
        sd = {**random_roberta_state_dict(seed=1, n_layer=layers, vocab=30522, max_pos=512, head=False,
                                          prefix="question_model."),
              **random_roberta_state_dict(seed=2, n_layer=layers, vocab=30522, max_pos=512, head=False, prefix="ctx_model.")}
        model = BiEncoder(type("A", (), {"num_hidden_layers": layers})())
        model.load_state_dict(sd)
        model = model.cuda()
        model.encoder_operand = fmt
        model.set_trainable(True, max_len=256)
        q, a = _batch(16, 256, 1, 30522, pad=0, cls=101), _batch(16, 256, 2, 30522, pad=0, cls=101)

        def ours():
            model.zero_grad(set_to_none=True)
            _in_batch(*model(q[0], q[1], a[0], a[1])).backward()

        def ours_forward():
            with torch.no_grad():
                _in_batch(*model(q[0], q[1], a[0], a[1]))

        orc = [EncoderOracle(sd, p, "bert", layers, 12, 0, 1e-12, device="cuda") for p in ("question_model.", "ctx_model.")]
        leaves = [t.requires_grad_(True) for o in orc for t in o.sd.values()]

        def oracle():
            for t in leaves:
                t.grad = None
            _in_batch(orc[0]._hidden_states(*q)[-1][:, 0], orc[1]._hidden_states(*a)[-1][:, 0]).backward()

        return ours, ours_forward, oracle, model
    cfg = roberta_base_config(num_hidden_layers=layers)
    sd = random_roberta_state_dict(seed=0, n_layer=layers)
    model = (RobertaDot_CLF_ANN_NLL_MultiChunk if workload == "maxp" else RobertaDot_NLL_LN)(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.cuda()
    model.encoder_operand = fmt
    model.set_trainable(True, max_len=128 if workload == "psg" else 512)
    if workload == "maxp":
        q, a, b = _batch(2, 64, 1, cfg.vocab_size), _batch(2, 2048, 2, cfg.vocab_size), _batch(2, 2048, 3, cfg.vocab_size)
    else:
        Ld = 128 if workload == "psg" else 512
        q, a, b = _batch(8, 64, 1, cfg.vocab_size), _batch(8, Ld, 2, cfg.vocab_size), _batch(8, Ld, 3, cfg.vocab_size)

    def ours():
        model.zero_grad(set_to_none=True)
        (loss,) = model(q[0], q[1], a[0], a[1], b[0], b[1])
        loss.backward()

    def ours_forward():   # the same loss without a graph: the inference forward
        with torch.no_grad():
            model(q[0], q[1], a[0], a[1], b[0], b[1])

    orc = RobertaDotOracle(sd, n_layer=layers, device="cuda")
    leaves = {k: v.requires_grad_(True) for k, v in orc.enc.sd.items()}
    head = [t.requires_grad_(True) for t in (orc.head_w, orc.head_b, orc.norm_g, orc.norm_b)]

    def emb(ids, mask):
        x = orc.enc._hidden_states(ids, mask)[-1][:, 0]
        return Fn.layer_norm(Fn.linear(x, head[0], head[1]), (768,), head[2], head[3], 1e-5)

    def chunks(ids, mask):
        B = ids.shape[0]
        return emb(ids.reshape(B * 4, 512), mask.reshape(B * 4, 512)).reshape(B, 4, 768)

    def oracle():
        for t in list(leaves.values()) + head:
            t.grad = None
        if workload == "maxp":
            _maxp_nll(emb(*q), chunks(*a), chunks(*b), a[1], b[1]).backward()
        else:
            _nll(emb(*q), emb(*a), emb(*b)).backward()

    return ours, ours_forward, oracle, model


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
    ap.add_argument("--workload", default="psg", choices=tuple(WORKLOADS))
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--fmt", default="fp16", choices=("fp16", "bf16"))
    ap.add_argument("--profile", action="store_true", help="also report our step's device time per kernel class")
    ap.add_argument("--dropout", action="store_true", help="time our step with and without dropout, alternating")
    ap.add_argument("--rounds", type=int, default=3, help="--dropout: rounds of (off, on)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train needs a GPU")
    ours, ours_forward, oracle, model = _setup(args.workload, args.layers, args.fmt)
    if args.dropout:
        return _dropout_ab(args, ours, model)

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
        "workload": f"{WORKLOADS[args.workload]}, {args.layers} layers, hidden 768",
        "operand_fmt": args.fmt, "step_ms_median": round(ours_ms, 3), "step_ms_min": round(ours_min, 3),
        "forward_only_ms_median": round(fwd_ms, 3), "oracle_fp32_eager_ms_median": round(orc_ms, 3), "oracle_fp32_eager_ms_min": round(orc_min, 3),
        "speedup_vs_oracle": round(orc_ms / ours_ms, 2), "gpu": name, "power_limit_w": float(power),
        "sm_clock_mhz_median": statistics.median(clk.samples) if clk.samples else None,
        "steps": args.steps, "warmup": args.warmup,
        "profile_ms_and_launches_per_step": profile}))


def _dropout_ab(args, ours, model):
    model.train()
    max_len = model._train_max_len
    rounds = {False: [], True: []}
    with ClockSampler() as clk:
        for _ in range(args.rounds):
            for on in (False, True):
                model.set_trainable(True, max_len=max_len, dropout=on)
                rounds[on].append(_time(ours, args.steps, args.warmup)[0])
    off, on = statistics.median(rounds[False]), statistics.median(rounds[True])
    profile = {}
    if args.profile:   # separate, untimed runs: device time per kernel class with dropout off and on
        for flag in (False, True):
            model.set_trainable(True, max_len=max_len, dropout=flag)
            _lib.profile_enable(True)
            _lib.profile_read(reset=True)
            for _ in range(args.steps):
                ours()
            torch.cuda.synchronize()
            profile["dropout" if flag else "no_dropout"] = {k: round(ms / args.steps, 3) for k, (ms, n) in
                                                            _lib.profile_read().items() if n}
            _lib.profile_enable(False)
    name, power = _smi("name,power.limit").split(", ")
    print(json.dumps({
        "workload": f"{WORKLOADS[args.workload]}, {args.layers} layers, hidden 768", "operand_fmt": args.fmt,
        "dropout": model._dropout if hasattr(model, "_dropout") else None,
        "step_ms_median_no_dropout": round(off, 3), "step_ms_median_dropout": round(on, 3),
        "dropout_cost_pct": round(100 * (on - off) / off, 2),
        "round_medians_no_dropout": [round(x, 3) for x in rounds[False]],
        "round_medians_dropout": [round(x, 3) for x in rounds[True]],
        "gpu": name, "power_limit_w": float(power),
        "sm_clock_mhz_median": statistics.median(clk.samples) if clk.samples else None,
        "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
        "profile_ms_per_step": profile or None}))


if __name__ == "__main__":
    main()
