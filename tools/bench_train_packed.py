"""Time one training step (forward + NLL loss + backward, 12 layers) with set_trainable(..., packed=False) (the padded
batch) and packed=True (the real tokens only), alternating the two modes in --rounds rounds of --steps steps within one
process, at the batch shapes of the reference's recipes and with lengths drawn from the repo's synthetic distributions:
  passage  rdot_nll, 8 triplets: queries padded to 64, lengths N(9, 3) clipped to [3, 64] (synthetic.py's MARCO-like
           queries); passages padded to 512, lengths N(76, 28) clipped to [5, 512] (its passages)
  maxp     rdot_nll_multi_chunk, 2 triplets: queries as above; documents of 4 x 512, lengths lognormal(log 1100, 0.8)
           clipped to [20, 2048] (tools/bench_packed.py's MaxP documents)
  dpr      the DPR BiEncoder, 16 (question, passage) pairs at 256 with in-batch negatives.  ASSUMED lengths: questions
           N(12, 4) clipped to [4, 256], passages N(160, 30) clipped to [20, 256] (tools/bench_packed.py's DPR passages)
  firstp   rdot_nll, 8 triplets at 512 (the control): queries as above, documents the MaxP lengths truncated to 512
The ids are random; every row's mask is a prefix, as the token caches make them.  The packed step includes its one
device-to-host copy of the lengths per encode.  Prints one JSON line per workload: median step time of each mode (and of
every round), the real-token fraction of the step's encodes, the training workspace bytes of one step in each mode, the
card's name, its power limit and the median SM clock sampled during the timed steps.

    python tools/bench_train_packed.py [--workload passage maxp dpr firstp] [--steps 10] [--warmup 3] [--rounds 3]
                                       [--fmt fp16|bf16] [--layers 12]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from ance_b200 import _lib  # noqa: E402
from ance_b200.models import BiEncoder, RobertaDot_CLF_ANN_NLL_MultiChunk, RobertaDot_NLL_LN  # noqa: E402
from ance_b200.synthetic import random_roberta_state_dict, roberta_base_config  # noqa: E402
from tools.bench_train import ClockSampler, _in_batch, _maxp_nll, _nll, _smi  # noqa: E402


def _lens(rng, kind, n, L):
    if kind == "query":
        x = rng.normal(9, 3, n).round().clip(3, L)
    elif kind == "passage":
        x = rng.normal(76, 28, n).round().clip(5, L)
    elif kind == "doc":
        x = np.round(rng.lognormal(np.log(1100), 0.8, n)).clip(20, 2048).clip(max=L)
    elif kind == "question":
        x = rng.normal(12, 4, n).round().clip(4, L)
    else:   # dpr passage
        x = rng.normal(160, 30, n).round().clip(20, L)
    return x.astype(np.int64)


def _batch(lens, L, vocab, pad, cls, seed):
    g = torch.Generator().manual_seed(seed)
    lens = torch.from_numpy(lens)
    ids = torch.randint(3, vocab, (len(lens), L), generator=g)
    mask = torch.arange(L)[None, :] < lens[:, None]
    ids = torch.where(mask, ids, torch.full_like(ids, pad))
    ids[:, 0] = cls
    return ids.cuda(), mask.long().cuda()


def _setup(workload, layers, fmt, rng):
    """-> (one training step, the model, [(encoder name, ids, mask)] of a step's encodes, the max_len to train with)."""
    if workload == "dpr":
        sd = {**random_roberta_state_dict(seed=1, n_layer=layers, vocab=30522, max_pos=512, head=False,
                                          prefix="question_model."),
              **random_roberta_state_dict(seed=2, n_layer=layers, vocab=30522, max_pos=512, head=False, prefix="ctx_model.")}
        model = BiEncoder(type("A", (), {"num_hidden_layers": layers})())
        model.load_state_dict(sd)
        model = model.cuda()
        model.encoder_operand = fmt
        q = _batch(_lens(rng, "question", 16, 256), 256, 30522, 0, 101, 1)
        a = _batch(_lens(rng, "dpr_passage", 16, 256), 256, 30522, 0, 101, 2)

        def step():
            model.zero_grad(set_to_none=True)
            _in_batch(*model(q[0], q[1], a[0], a[1])).backward()

        return step, model, [("question", *q), ("ctx", *a)], 256
    cfg = roberta_base_config(num_hidden_layers=layers)
    sd = random_roberta_state_dict(seed=0, n_layer=layers)
    model = (RobertaDot_CLF_ANN_NLL_MultiChunk if workload == "maxp" else RobertaDot_NLL_LN)(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.cuda()
    model.encoder_operand = fmt
    V = cfg.vocab_size
    if workload == "maxp":
        q = _batch(_lens(rng, "query", 2, 64), 64, V, 1, 0, 1)
        a, b = (_batch(_lens(rng, "doc", 2, 2048), 2048, V, 1, 0, s) for s in (2, 3))

        def step():
            model.zero_grad(set_to_none=True)
            _maxp_nll(model.query_emb(*q), model.body_emb(*a), model.body_emb(*b), a[1], b[1]).backward()

        chunks = [(x[0].reshape(-1, 512), x[1].reshape(-1, 512)) for x in (a, b)]
        return step, model, [("roberta", *q)] + [("roberta", *c) for c in chunks], 512
    q = _batch(_lens(rng, "query", 8, 64), 64, V, 1, 0, 1)
    kind = "passage" if workload == "passage" else "doc"
    a, b = (_batch(_lens(rng, kind, 8, 512), 512, V, 1, 0, s) for s in (2, 3))

    def step():
        model.zero_grad(set_to_none=True)
        (loss,) = model(q[0], q[1], a[0], a[1], b[0], b[1])
        loss.backward()

    return step, model, [("roberta", *q), ("roberta", *a), ("roberta", *b)], 512


def _workspace(model, encodes, packed):
    """Training workspace bytes of one step's encodes (all-padding MaxP chunks: one dense 512-token row per encode)."""
    total = 0
    lib = _lib.load()
    cache = model.__dict__["_enc_cache"]
    for name, ids, mask in encodes:
        h = cache[name][1].h
        B, L = ids.shape
        n = C.c_size_t()
        lens = mask.sum(1).to(torch.int32).cpu()
        if packed:
            real = lens[lens > 0].contiguous()
            _lib.check(lib.ance_encoder_train_workspace_packed(h, real.data_ptr(), len(real), L, C.byref(n)))
            total += n.value
            if len(real) < B:
                _lib.check(lib.ance_encoder_train_workspace(h, 1, L, C.byref(n)))
                total += n.value
        else:
            _lib.check(lib.ance_encoder_train_workspace(h, B, L, C.byref(n)))
            total += n.value
    return total


def _time(step, steps):
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        step()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=["passage", "maxp", "dpr", "firstp"],
                    choices=("passage", "maxp", "dpr", "firstp"))
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--fmt", default="fp16", choices=("fp16", "bf16"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_train_packed.py times the GPU: no CUDA device"
    name, power = _smi("name"), _smi("power.limit")
    for wl in args.workload:
        rng = np.random.default_rng(7)
        step, model, encodes, max_len = _setup(wl, args.layers, args.fmt, rng)
        for packed in (False, True):   # warm up both modes (module loads, workspace sizes)
            model.set_trainable(True, max_len=max_len, packed=packed)
            for _ in range(args.warmup):
                step()
        torch.cuda.synchronize()
        rounds = {"dense": [], "packed": []}
        with ClockSampler() as clk:
            for _ in range(args.rounds):
                for mode in ("dense", "packed"):
                    model.set_trainable(True, max_len=max_len, packed=mode == "packed")
                    rounds[mode].append(_time(step, args.steps))
        real = sum(int(m.sum()) for _, _, m in encodes)
        slots = sum(m.numel() for _, _, m in encodes)
        med = {k: statistics.median(v) for k, v in rounds.items()}
        print(json.dumps({
            "workload": wl, "layers": args.layers, "fmt": args.fmt,
            "step_ms_dense": round(med["dense"], 2), "step_ms_packed": round(med["packed"], 2),
            "speedup": round(med["dense"] / med["packed"], 2),
            "rounds_ms": {k: [round(x, 2) for x in v] for k, v in rounds.items()},
            "real_token_fraction": round(real / slots, 4),
            "workspace_bytes_dense": _workspace(model, encodes, False),
            "workspace_bytes_packed": _workspace(model, encodes, True),
            "gpu": name, "power_limit_w": power,
            "sm_clock_mhz_median": statistics.median(clk.samples) if clk.samples else None,
        }), flush=True)
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
