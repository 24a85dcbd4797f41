"""Host-side rows of SURVEY.md par. 8(f), timed on this machine's CPU cores (no GPU involved):
  row 1  negative sampling + file emission: ance_b200.postprocess (vectorised) vs the reference-style per-query loop
         (oracle.refresh_oracle.generate_negatives, the restatement of run_ann_data_gen.py:339-400)
  row 2  token-cache reading: ance_b200.data.StridedBatchReader (bulk memmap gather) vs the reference-style
         StreamingDataset(cache, GetProcessingFn) record iterator
  (e)    host k-way merge of per-shard top-k (csrc/merge.cpp)
Writes one JSON object to stdout."""
import argparse
import json
import os
import random
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from ance_b200 import postprocess  # noqa: E402
from ance_b200.data import EmbeddingCache, GetProcessingFn, StreamingDataset, StridedBatchReader  # noqa: E402
from oracle import refresh_oracle  # noqa: E402


def bench_negatives(nq, k, n_p, loop_sample):
    rng = np.random.default_rng(0)
    I = rng.integers(0, n_p, size=(nq, k), dtype=np.int64)
    q2id = np.arange(nq, dtype=np.int64)
    p2id = np.arange(n_p, dtype=np.int64)
    pos = {int(q): int(I[q, rng.integers(0, k)]) for q in range(nq)}
    t0 = time.perf_counter()
    negs, _, _ = postprocess.generate_negatives(q2id, p2id, pos, I, 20, False, sampler="fast", seed=0)
    t_cold = time.perf_counter() - t0          # first call in the process: page faults of the temporaries
    t0 = time.perf_counter()
    negs, _, _ = postprocess.generate_negatives(q2id, p2id, pos, I, 20, False, sampler="fast", seed=0)
    t_fast = time.perf_counter() - t0
    with tempfile.TemporaryDirectory() as td:
        t0 = time.perf_counter()
        postprocess.write_training_data(os.path.join(td, "ann_training_data_0"), q2id, pos, negs)
        t_write = time.perf_counter() - t0
    m = loop_sample
    t0 = time.perf_counter()
    refresh_oracle.generate_negatives(q2id[:m], p2id, pos, I[:m], set(q2id[:m].tolist()), 20, False, random.Random(0))
    t_loop = (time.perf_counter() - t0) * nq / m
    return {"queries": nq, "topk": k, "vectorised_s": t_fast, "vectorised_first_call_s": t_cold, "write_file_s": t_write,
            "reference_style_loop_s_extrapolated": t_loop, "loop_sample": m, "speedup": t_loop / t_fast}


def bench_reader(n, L, loop_sample):
    rng = np.random.default_rng(1)
    lens = rng.integers(8, L + 1, size=n)
    ids = rng.integers(3, 50000, size=(n, L), dtype=np.int32)
    with tempfile.TemporaryDirectory() as td:
        base = os.path.join(td, "passages")
        refresh_oracle.write_cache(base, lens, ids)
        cache = EmbeddingCache(base)
        with cache:
            t0 = time.perf_counter()
            tot = 0
            for b_ids, b_lens, b_idx in StridedBatchReader(cache, 592, rank=0, world_size=1, pin=False):
                tot += int(b_ids.shape[0])
            t_bulk = time.perf_counter() - t0
            assert tot == n
            args = argparse.Namespace(max_seq_length=L, max_query_length=L)
            t0 = time.perf_counter()
            for j, rec in enumerate(StreamingDataset(cache, GetProcessingFn(args, query=False), distributed=False)):
                if j + 1 >= loop_sample:
                    break
            t_rec = (time.perf_counter() - t0) * n / loop_sample
    return {"records": n, "L": L, "bulk_reader_s": t_bulk, "bulk_records_per_s": n / t_bulk,
            "per_record_iterator_s_extrapolated": t_rec, "per_record_records_per_s": n / t_rec, "loop_sample": loop_sample}


def bench_merge(nq, k, shards):
    from ance_b200.search import merge_topk_host
    rng = np.random.default_rng(2)
    Ds = [np.sort(rng.standard_normal((nq, k)).astype(np.float32), axis=1)[:, ::-1].copy() for _ in range(shards)]
    Is = [rng.integers(0, 1 << 40, size=(nq, k), dtype=np.int64) for _ in range(shards)]
    merge_topk_host(Ds, Is, k)   # first call: output page faults
    t0 = time.perf_counter()
    merge_topk_host(Ds, Is, k)
    dt = time.perf_counter() - t0
    t0 = time.perf_counter()
    merge_topk_host(Ds, Is, k, 1)
    d1 = time.perf_counter() - t0
    return {"queries": nq, "topk": k, "shards": shards, "seconds": dt, "queries_per_s": nq / dt, "single_thread_seconds": d1}


def bench_answer_filter(n_q, topk, n_p):
    """row 4: DPR answer-string filter of `validate` (run_ann_data_gen_dpr.py:281-340): n_q questions x topk passages."""
    from ance_b200.dpr_utils import AnswerMatcher, has_answer
    rng = np.random.default_rng(3)
    vocab = ["w%d" % i for i in range(5000)]
    texts = {i: (" ".join(vocab[j] for j in rng.integers(0, 5000, size=100)), "t") for i in range(n_p)}
    answers = [[" ".join(vocab[j] for j in rng.integers(0, 5000, size=2))] for _ in range(n_q)]
    I = rng.zipf(1.3, size=(n_q, topk)) % n_p          # popular passages are retrieved for many questions
    m = AnswerMatcher(texts)
    t0 = time.perf_counter()
    hits = sum(m.has_answer(answers[q], int(I[q, j])) for q in range(n_q) for j in range(topk))
    t_cached = time.perf_counter() - t0
    sample = max(1, n_q // 10)
    t0 = time.perf_counter()
    hits_ref = sum(has_answer(answers[q], texts[int(I[q, j])][0]) for q in range(sample) for j in range(topk))
    t_ref = (time.perf_counter() - t0) * n_q / sample
    return {"questions": n_q, "topk": topk, "distinct_passages": int(len(np.unique(I))), "cached_matcher_s": t_cached,
            "reference_style_s_extrapolated": t_ref, "speedup": t_ref / t_cached, "hits": int(hits), "hits_sample_ref": int(hits_ref)}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--nq", type=int, default=100000)
    ap.add_argument("--records", type=int, default=200000)
    a = ap.parse_args()
    out = {"cpu_count": os.cpu_count(),
           "row1_negatives": bench_negatives(a.nq, 200, 8841823, 2000),
           "row2_reader": bench_reader(a.records, 128, 20000)}
    out["row4_dpr_answer_filter"] = bench_answer_filter(3610, 100, 200000)
    try:
        out["merge_8_shards"] = bench_merge(a.nq, 200, 8)
    except Exception as e:  # the C ABI library is needed for the merge
        out["merge_8_shards"] = {"error": str(e)}
    print(json.dumps(out, indent=1))
