"""Host index (fp32 rows in pinned host memory) against the device index, on one GPU.

(a) Seeded clustered LayerNorm-like rows (tools/bringup_search.make_data), 8,841,823 x 768, fp16 operands, one device
    index and one host index over the same rows, searched alternately.  Cases: 2,368 and 18,944 queries at k = 200,
    18,944 at k = 1000.  Per case and mode: ms per search (CUDA events, mean of --iters), device ms of the coarse pass
    and of the rescoring (ance_profile_read, a separate profiled search), candidates rescored, rows fetched from host
    memory, the GB they make and the PCIe rate that implies over the host rescoring's device time, memory() of both
    indexes, torch.equal of D and I between the modes, and the first and last 32 queries of every query block (k > 512:
    blocks of at most 16,384) of the host index's answer against its exact=True.  Also the host index's add (D2H) and prepare (H2D) times.
(b) A host index of 21,015,324 rows (DPR's corpus), generated on the GPU in blocks and added block by block: add and
    prepare time, searches at DPR's shapes (58,880 queries at k = 200; 3,610 and 11,313 at k = 100), memory(), and the
    first and last 32 queries of every query block compared bit for bit with exact=True (the brute force copies the rows
    H2D once per query batch), with the time that takes.  Skipped, with the reason, when MemAvailable is below the 65 GB of pinned rows it needs.
The card's name, power limit and SM clock are read in the same run.  One JSON line per record.

    python tools/bench_host_rows.py [--iters 2] [--parts ab] [--out FILE]
"""
import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402

from ance_b200 import _lib  # noqa: E402
from ance_b200.search import IndexFlatIP  # noqa: E402
from tools.bench_large_k import block_edges, equals_exact, gpu_info  # noqa: E402
from tools.bringup_search import make_data  # noqa: E402

D = 768
ROWS_A = 8841823
CASES_A = [(2368, 200), (18944, 200), (18944, 1000)]
ROWS_B = 21015324
CASES_B = [(58880, 200), (3610, 100), (11313, 100)]


def mem_available() -> int:
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            return int(line.split()[1]) * 1024
    return 0


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def search_ms(idx, q, k, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        Dv, Iv = idx.search_device(q, k)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, Dv, Iv


def profiled(idx, q, k):
    _lib.profile_enable(True)
    _lib.profile_read(reset=True)
    idx.search_device(q, k)
    prof = _lib.profile_read(reset=True)
    _lib.profile_enable(False)
    return {c: round(prof[c][0], 3) for c in ("quantize", "coarse_search", "rescore", "exact")}


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        out.write(line + "\n")
        out.flush()


def part_a(a, dev, out):
    P, Q = make_data(ROWS_A, max(nq for nq, _ in CASES_A), D, "clustered", dev)
    di = IndexFlatIP(D, operand="fp16", storage=P)
    di.add(P)
    di.prepare()
    hi = IndexFlatIP(D, capacity=ROWS_A, operand="fp16", rows="host")
    t_add = timed(lambda: hi.add(P))
    t_prep = timed(hi.prepare)
    gb = ROWS_A * D * 4 / 1e9
    emit({"part": "a", "what": "host index build", "rows": ROWS_A, "add_s": round(t_add, 3),
          "add_d2h_GBps": round(gb / t_add, 1), "prepare_s": round(t_prep, 3),
          "prepare_h2d_GBps_2_passes": round(2 * gb / t_prep, 1), "gpu": gpu_info()}, out)
    for nq, k in CASES_A:
        q = Q[:nq].contiguous()
        for idx in (di, hi):   # warm-up (workspace growth) of both
            idx.search_device(q, k)
        ms = {"device": [], "host": []}
        for _ in range(a.iters):   # alternate the modes
            for name, idx in (("device", di), ("host", hi)):
                m, Dv, Iv = search_ms(idx, q, k, 1)
                ms[name].append(m)
        Dd, Id = di.search_device(q, k)
        std = di.stats()
        Dh, Ih = hi.search_device(q, k)
        sth, fetched = hi.stats(), hi.last_fetched()
        prof_d, prof_h = profiled(di, q, k), profiled(hi, q, k)
        edges = block_edges(nq, k)
        exact_ok = equals_exact(hi, q, k, Dh, Ih, edges)
        fetched_gb = fetched * D * 4 / 1e9
        emit({"part": "a", "rows": ROWS_A, "nq": nq, "k": k, "operand": "fp16",
              "device_ms": round(sum(ms["device"]) / len(ms["device"]), 3),
              "host_ms": round(sum(ms["host"]) / len(ms["host"]), 3),
              "device_kernel_ms": prof_d, "host_kernel_ms": prof_h,
              "n_candidates": sth["n_candidates"], "n_candidates_device": std["n_candidates"],
              "n_splits": sth["n_splits"], "n_tier2": sth["n_tier2"], "n_uncertified": sth["n_uncertified"],
              "fetched_rows": fetched, "fetched_GB": round(fetched_gb, 3),
              "implied_pcie_GBps": round(fetched_gb / (prof_h["rescore"] / 1e3), 1) if prof_h["rescore"] else None,
              "memory_device_index": di.memory(), "memory_host_index": hi.memory(),
              "equal_D_I": bool(torch.equal(Dd, Dh) and torch.equal(Id, Ih)), "exact_block_edges": len(edges),
              "exact_block_edges_bitexact": exact_ok, "gpu": gpu_info()}, out)
    del di, hi, P, Q
    torch.cuda.empty_cache()


def gen_block(n, seed, dev, cent):
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    x = torch.randn(n, D, device=dev, generator=g)
    x = 0.5 * x + 0.5 * cent[torch.randint(0, 1024, (n,), device=dev, generator=g)]
    return (x - x.mean(1, keepdim=True)) / x.std(1, keepdim=True, unbiased=False)


def part_b(a, dev, out):
    need = ROWS_B * D * 4 + (8 << 30)
    if mem_available() < need:
        emit({"part": "b", "skipped": f"MemAvailable {mem_available() / 2**30:.1f} GiB < {need / 2**30:.1f} GiB needed "
                                      "for the pinned rows"}, out)
        return
    g = torch.Generator(device=dev)
    g.manual_seed(7)
    cent = torch.randn(1024, D, device=dev, generator=g)
    t0 = time.perf_counter()
    hi = IndexFlatIP(D, capacity=ROWS_B, operand="fp16", rows="host")
    t_alloc = time.perf_counter() - t0
    blk = 1 << 21
    t_add = 0.0
    for s in range(0, ROWS_B, blk):
        x = gen_block(min(blk, ROWS_B - s), 1000 + s // blk, dev, cent)
        t_add += timed(lambda: hi.add(x))
    t_prep = timed(hi.prepare)
    gb = ROWS_B * D * 4 / 1e9
    emit({"part": "b", "what": "host index build", "rows": ROWS_B, "pin_alloc_s": round(t_alloc, 3),
          "add_s": round(t_add, 3), "add_d2h_GBps": round(gb / t_add, 1), "prepare_s": round(t_prep, 3),
          "prepare_h2d_GBps_2_passes": round(2 * gb / t_prep, 1), "memory": hi.memory(), "gpu": gpu_info()}, out)
    Q = gen_block(max(nq for nq, _ in CASES_B), 4321, dev, cent)
    for nq, k in CASES_B:
        q = Q[:nq].contiguous()
        hi.search_device(q, k)   # warm-up
        ms, Dh, Ih = search_ms(hi, q, k, 1)
        st, fetched = hi.stats(), hi.last_fetched()
        prof = profiled(hi, q, k)
        edges = block_edges(nq, k)
        res = {}
        t_exact = timed(lambda: res.update(ok=equals_exact(hi, q, k, Dh, Ih, edges)))
        fetched_gb = fetched * D * 4 / 1e9
        emit({"part": "b", "rows": ROWS_B, "nq": nq, "k": k, "operand": "fp16", "host_ms": round(ms, 3),
              "qps": round(nq / ms * 1e3, 1), "kernel_ms": prof, "n_candidates": st["n_candidates"],
              "n_splits": st["n_splits"], "n_tier2": st["n_tier2"], "n_uncertified": st["n_uncertified"],
              "fetched_rows": fetched, "fetched_GB": round(fetched_gb, 3),
              "implied_pcie_GBps": round(fetched_gb / (prof["rescore"] / 1e3), 1) if prof["rescore"] else None,
              "memory": hi.memory(), "exact_block_edges": len(edges), "exact_block_edges_s": round(t_exact, 3),
              "exact_block_edges_bitexact": res["ok"], "gpu": gpu_info()}, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--parts", default="ab", choices=["ab", "a", "b"])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_host_rows needs a CUDA device")
    dev = torch.device("cuda:0")
    out = open(a.out, "a") if a.out else None
    if "a" in a.parts:
        part_a(a, dev, out)
    if "b" in a.parts:
        part_b(a, dev, out)


if __name__ == "__main__":
    main()
