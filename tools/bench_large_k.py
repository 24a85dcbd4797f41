"""Large-k flat inner-product search (512 < k <= 2048) at full corpus size, on one GPU.

Seeded clustered LayerNorm-like rows (SURVEY.md §8d; tools/bringup_search.make_data), 8,841,823 x 768, fp16 operands.
One JSON line per case:
  dev-small     6,980 queries at k = 100 (the refresh's dev search) and k = 1000 (top-1000 full-rank evaluation)
  driver block  18,944 queries (one block of the driver's search) at k = 200, 500, 1000, 2048
Per case: ms per search and queries/s (CUDA events, mean of --iters searches after a warm-up), the search statistics
(kprime, n_splits, n_tier2, n_uncertified, n_candidates), device ms per kernel class from ance_profile_read (a separate
profiled search), the workspace the search allocated (device memory in use after its first search on a fresh index
minus before), and bit-exact agreement of the first 64 queries with search_device(..., exact=True).  The card's name,
power limit and SM clock are read in the same run.

    python tools/bench_large_k.py [--rows 8841823] [--iters 3] [--out FILE]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402

from ance_b200 import _lib  # noqa: E402
from ance_b200.search import IndexFlatIP  # noqa: E402
from tools.bringup_search import make_data  # noqa: E402

CASES = [(6980, 100), (6980, 1000), (18944, 200), (18944, 500), (18944, 1000), (18944, 2048)]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:   # the numbers still stand, but without the card they are incomplete
        return {"error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=8841823)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_large_k needs a CUDA device")
    dev = torch.device("cuda:0")
    P, Q = make_data(a.rows, max(nq for nq, _ in CASES), 768, "clustered", dev)
    out = open(a.out, "a") if a.out else None
    for nq, k in CASES:
        # a fresh index over the same rows per case, so that the workspace measured is this case's alone
        idx = IndexFlatIP(768, operand="fp16", storage=P)
        idx.add(P)
        idx.prepare()
        q = Q[:nq].contiguous()
        # the result tensors come from torch's caching allocator: reserve them first, so only the library's workspace counts
        D_, I_ = torch.empty((nq, k), device=dev), torch.empty((nq, k), dtype=torch.int64, device=dev)
        del D_, I_
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(dev)[0]
        D, I = idx.search_device(q, k)
        torch.cuda.synchronize()
        workspace = free0 - torch.cuda.mem_get_info(dev)[0]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            D, I = idx.search_device(q, k)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.iters
        info = gpu_info()
        st = idx.stats()
        _lib.profile_enable(True)
        _lib.profile_read(reset=True)
        idx.search_device(q, k)
        prof = _lib.profile_read(reset=True)
        _lib.profile_enable(False)
        De, Ie = idx.search_device(q[:64], k, exact=True)
        torch.cuda.synchronize()
        exact_ok = bool((Ie == I[:64]).all().item() and (De.view(torch.int32) == D[:64].view(torch.int32)).all().item())
        rec = {"case": "dev-small" if nq == 6980 else "driver-block", "rows": a.rows, "nq": nq, "k": k, "operand": "fp16",
               "ms": round(ms, 3), "qps": round(nq / ms * 1e3, 1),
               "kprime": st["kprime"], "n_splits": st["n_splits"], "n_tier2": st["n_tier2"],
               "n_uncertified": st["n_uncertified"], "n_candidates": st["n_candidates"],
               "device_ms": {c: round(prof[c][0], 3) for c in ("quantize", "coarse_search", "rescore", "exact")},
               "workspace_bytes": int(workspace), "exact_slice_64_bitexact": exact_ok, "gpu": info}
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()
        del idx, D, I, De, Ie
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
