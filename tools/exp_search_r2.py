"""Search experiments on one GPU (results appended to the JSONL file OUT below):

  certify   per distribution (ance_b200.synthetic.synth_index_rows kinds) x operand format, default k': how many queries
            need tier 2 / tier 3, max eps, and what the whole search costs — the certification-cliff question of VERDICT r1
  pace      the soft barrier between sweeping CTA pairs on/off at nq = one wave and several waves: coarse ms, TFLOP/s

  python tools/exp_search_r2.py certify 8841823 18944 layernorm_clustered,iid,heavy_tail,near_duplicate,dpr
  python tools/exp_search_r2.py pace 8841823 18944,75776
"""
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402

from ance_b200 import _lib  # noqa: E402
from ance_b200.search import IndexFlatIP  # noqa: E402
from ance_b200.synthetic import synth_index_rows  # noqa: E402

OUT = ROOT / "gpurun_out" / "exp_search_r2.jsonl"
DIM = 768


def build(N, kind, operand, dev):
    idx = IndexFlatIP(DIM, capacity=N, device=dev, operand=operand)
    for x in synth_index_rows(N, DIM, dev, 1234, kind):
        idx.add(x)
    torch.cuda.synchronize()
    return idx


def queries(nq, kind, dev):
    return torch.cat(list(synth_index_rows(nq, DIM, dev, 4321, kind))).contiguous()


def timed_search(idx, Q, k):
    idx.search_device(Q, k)
    torch.cuda.synchronize()
    _lib.profile_read(reset=True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    idx.search_device(Q, k)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), _lib.profile_read(reset=True), idx.stats()


def emit(rec):
    print(json.dumps(rec), flush=True)
    with open(OUT, "a") as f:
        f.write(json.dumps(rec) + "\n")


def certify(N, nq, kinds):
    dev = torch.device("cuda:0")
    for kind in kinds:
        Q = queries(nq, kind, dev)
        k = 100 if kind == "dpr" else 200
        for operand in ("fp16", "bf16"):
            idx = build(N, kind, operand, dev)
            for kp in (0,) if operand == "bf16" else (0, 224 if k == 200 else 128):
                idx.set_param("kprime", kp)
                ms, prof, st = timed_search(idx, Q, k)
                emit({"exp": "certify", "N": N, "nq": nq, "kind": kind, "operand": operand, "k": k, "kprime": st["kprime"],
                      "n_tier2": st["n_tier2"], "n_brute_force": st["n_uncertified"], "max_eps": st["max_eps"],
                      "candidates_per_query": st["n_candidates"] / nq, "ms": ms, "qps": nq / ms * 1e3,
                      "coarse_ms": prof["coarse_search"][0], "coarse_launches": prof["coarse_search"][1],
                      "rescore_ms": prof["rescore"][0], "exact_ms": prof["exact"][0]})
            del idx
            torch.cuda.empty_cache()


def pace(N, nqs, windows=(0, 16, 32, 64, 128)):
    dev = torch.device("cuda:0")
    idx = build(N, "layernorm_clustered", "fp16", dev)
    Qall = queries(max(nqs), "layernorm_clustered", dev)
    for nq in nqs:
        Q = Qall[:nq].contiguous()
        for window in windows:
            idx.set_param("pace_window", window)
            ms, prof, st = timed_search(idx, Q, 200)
            c = prof["coarse_search"][0]
            emit({"exp": "pace", "N": N, "nq": nq, "pace_window": window, "ms": ms, "qps": nq / ms * 1e3, "coarse_ms": c,
                  "coarse_tflops": 2.0 * nq * N * DIM / c / 1e9, "rescore_ms": prof["rescore"][0], "n_tier2": st["n_tier2"],
                  "candidates_per_query": st["n_candidates"] / nq})


if __name__ == "__main__":
    _lib.profile_enable(True)
    if sys.argv[1] == "certify":
        certify(int(sys.argv[2]), int(sys.argv[3]), sys.argv[4].split(","))
    elif sys.argv[1] == "pace1":   # one configuration (the default window), short enough to sit under ncu
        pace(int(sys.argv[2]), [int(x) for x in sys.argv[3].split(",")], windows=(16,))
    else:
        pace(int(sys.argv[2]), [int(x) for x in sys.argv[3].split(",")])
