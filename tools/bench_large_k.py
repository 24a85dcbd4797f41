"""Large-k flat inner-product search (512 < k <= 2048) at full corpus size, on one GPU.

Seeded clustered LayerNorm-like rows (SURVEY.md §8d; tools/bringup_search.make_data), 8,841,823 x 768, fp16 operands.
One JSON line per case:
  dev-small     6,980 queries at k = 100 (the refresh's dev search) and k = 1000 (top-1000 full-rank evaluation)
  driver block  18,944 queries (one block of the driver's search) at k = 200, 500, 1000, 2048
Per case: ms per search and queries/s (CUDA events, mean of --iters searches after a warm-up), the search statistics
(kprime, n_splits, n_tier2, n_uncertified, n_candidates), device ms per kernel class from ance_profile_read (a separate
profiled search), the workspace the search allocated (device memory in use after its first search on a fresh index
minus before), and bit-exact agreement with search_device(..., exact=True) of the first and last 32 queries of every
query block (k > 512: blocks of at most 16,384; otherwise the call is one block).  The card's name, power limit and SM
clock are read in the same run.

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
WIDE_QBLOCK = 16384   # search.cu kWideQBlock


def block_edges(nq, k, edge=32):
    """Query numbers of the first and last `edge` queries of every block ance_index_search splits nq into (k > 512:
    equal blocks of at most 16,384 rounded up to the 256-query tile; otherwise one block)."""
    qb = nq
    if k > 512:
        n_blocks = -(-nq // WIDE_QBLOCK)
        qb = min(WIDE_QBLOCK, -(-(-(-nq // n_blocks)) // 256) * 256)
    rows = set()
    for b0 in range(0, nq, qb):
        b1 = min(nq, b0 + qb)
        rows |= set(range(b0, min(b1, b0 + edge))) | set(range(max(b0, b1 - edge), b1))
    return sorted(rows)


def equals_exact(idx, q, k, D, I, rows):
    """D / I of `rows` bit for bit equal to the brute force's answer for those queries."""
    r = torch.as_tensor(rows, device=q.device)
    De, Ie = idx.search_device(q[r].contiguous(), k, exact=True)
    return bool(torch.equal(Ie, I[r]) and torch.equal(De.view(torch.int32), D[r].view(torch.int32)))


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
        edges = block_edges(nq, k)
        exact_ok = equals_exact(idx, q, k, D, I, edges)
        rec = {"case": "dev-small" if nq == 6980 else "driver-block", "rows": a.rows, "nq": nq, "k": k, "operand": "fp16",
               "ms": round(ms, 3), "qps": round(nq / ms * 1e3, 1),
               "kprime": st["kprime"], "n_splits": st["n_splits"], "n_tier2": st["n_tier2"],
               "n_uncertified": st["n_uncertified"], "n_candidates": st["n_candidates"],
               "device_ms": {c: round(prof[c][0], 3) for c in ("quantize", "coarse_search", "rescore", "exact")},
               "workspace_bytes": int(workspace), "exact_block_edges": len(edges), "exact_block_edges_bitexact": exact_ok,
               "gpu": info}
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()
        del idx, D, I
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
