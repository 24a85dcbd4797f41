"""Parity of the sm_90a flat inner-product search with the CPU oracle (bit-exact: int64 labels and
fp32 scores), through the C ABI (ance_b200.search.IndexFlatIP -> ctypes -> libance_b200.so)."""
import os

import numpy as np
import pytest
import torch

from oracle import flat_ip_oracle

pytestmark = pytest.mark.gpu


def _ln_rows(rng, n, d, clustered=True):
    x = rng.standard_normal((n, d)).astype(np.float32)
    if clustered:
        cent = np.random.default_rng(7).standard_normal((64, d)).astype(np.float32)
        x = 0.5 * x + 0.5 * cent[rng.integers(0, 64, size=n)]
    x = (x - x.mean(1, keepdims=True)) / x.std(1, keepdims=True)
    return np.ascontiguousarray(x.astype(np.float32))


def _index(P, operand="auto", **params):
    from ance_b200.search import IndexFlatIP
    idx = IndexFlatIP(P.shape[1], capacity=max(1, P.shape[0]), operand=operand)
    idx.add(P)
    for k, v in params.items():
        idx.set_param(k, v)
    return idx


def test_golden_kat(golden_dir):
    g = np.load(os.path.join(golden_dir, "search_kat.npz"))
    rng = np.random.default_rng(int(g["seed"]))
    P = rng.standard_normal((3000, 64)).astype(np.float32)
    P[1500:1510] = P[10:20]
    Q = rng.standard_normal((16, 64)).astype(np.float32)
    Q[0] = P[12] * 2
    for operand in ("auto", "bf16", "fp16"):
        D, I = _index(P, operand).search(Q, 20)
        assert (I == g["I"]).all() and (D == g["D"]).all()


@pytest.mark.parametrize("operand", ["bf16", "fp16"])
@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("k", [10, 100, 200])
def test_seeded_parity(operand, cta_group, k):
    rng = np.random.default_rng(1234)
    P = _ln_rows(rng, 60000, 768)
    Q = _ln_rows(np.random.default_rng(4321), 300, 768)
    idx = _index(P, operand, cta_group=cta_group)
    D, I = idx.search(Q, k)
    Do, Io = flat_ip_oracle.search(P, Q, k)
    assert (I == Io).all(), f"{(I != Io).any(1).sum()} queries differ"
    assert (D == Do).all()
    st = idx.stats()
    assert st["nq"] == 300 and st["kprime"] >= k
    # scores within 1e-3 relative of a plain fp32 sgemm (the faiss arithmetic), as north_star asks
    S = Q @ P.T
    ref = np.take_along_axis(S, I, axis=1)
    assert np.abs(D - ref).max() <= 1e-3 * np.abs(ref).max()


def test_default_topk_training_500():
    """`--topk_training` defaults to 500 (run_ann_data_gen.py:556-560): the 2048-entry reservoir path (k' = 992)."""
    rng = np.random.default_rng(21)
    P = _ln_rows(rng, 50000, 768)
    Q = _ln_rows(np.random.default_rng(22), 130, 768)
    for k in (300, 500):
        idx = _index(P)
        D, I = idx.search(Q, k)
        Do, Io = flat_ip_oracle.search(P, Q, k)
        assert (I == Io).all() and (D == Do).all()
        assert idx.stats()["kprime"] >= k


def test_duplicates_and_ties_are_ordered_by_row():
    rng = np.random.default_rng(5)
    P = _ln_rows(rng, 20000, 768)
    P[10000:10050] = P[0:50]           # exact duplicates -> exact score ties
    Q = _ln_rows(np.random.default_rng(6), 64, 768)
    Q[:50] = P[0:50] + 0.01 * Q[:50]   # queries whose best neighbours are the duplicated rows
    D, I = _index(P).search(Q, 20)
    Do, Io = flat_ip_oracle.search(P, Q, 20)
    assert (I == Io).all() and (D == Do).all()
    for q in range(50):
        a, b = np.where(I[q] == q)[0], np.where(I[q] == 10000 + q)[0]
        assert len(a) == 1 and len(b) == 1 and b[0] == a[0] + 1  # tie: smaller row first


def test_uncertified_queries_fall_back_to_exact():
    """Thousands of EXACTLY equal rows at the top of every ranking: no 16-bit pass can separate them (thr == s_k), the
    tier-2 pass from the threshold s_k - eps lets all of them through and its reservoir overflows, so the exact
    brute-force path must produce the oracle's answer (ties in ascending row order)."""
    rng = np.random.default_rng(8)
    base = _ln_rows(rng, 1, 768)
    P = _ln_rows(np.random.default_rng(80), 16384, 768)
    P[::2] = base                                      # 8192 identical rows, interleaved with ordinary ones
    Q = (base * 1.0 + 0.05 * _ln_rows(np.random.default_rng(9), 32, 768)).astype(np.float32)   # queries near the duplicated row
    idx = _index(P)
    D, I = idx.search(Q, 50)
    Do, Io = flat_ip_oracle.search_bruteforce(P, Q, 50)
    assert (I == Io).all() and (D == Do).all()
    assert (I[:, :50] % 2 == 0).all() and (np.diff(I, axis=1) > 0).all()     # the duplicates, smallest rows first
    assert idx.stats()["n_uncertified"] > 0


def test_edges_empty_small_and_offsets():
    rng = np.random.default_rng(10)
    P = _ln_rows(rng, 37, 768, clustered=False)
    Q = _ln_rows(np.random.default_rng(11), 5, 768, clustered=False)
    idx = _index(P)
    D, I = idx.search(Q, 50)  # fewer rows than k: faiss pads with -1 / lowest float
    Do, Io = flat_ip_oracle.search_bruteforce(P, Q, 50)
    assert (I == Io).all() and (D == Do).all() and (I[:, 37:] == -1).all()
    D0, I0 = idx.search(Q[:0], 5)
    assert D0.shape == (0, 5) and I0.shape == (0, 5)
    from ance_b200.search import IndexFlatIP
    empty = IndexFlatIP(768)
    De, Ie = empty.search(Q, 3)
    assert (Ie == -1).all()
    # row_offset (per-shard global numbering) on the tensor-core path
    P2 = _ln_rows(rng, 5000, 768)
    idx2 = _index(P2)
    Dd, Id = idx2.search_device(torch.from_numpy(Q).cuda(), 10, row_offset=123456)
    _, Io2 = flat_ip_oracle.search(P2, Q, 10)
    assert (Id.cpu().numpy() == Io2 + 123456).all()
    with pytest.raises(ValueError):
        idx2.search(np.zeros((2, 64), dtype=np.float32), 3)
    with pytest.raises(TypeError):
        idx2.search(np.zeros((2, 768), dtype=np.float64), 3)


def test_exact_path_equals_oracle():
    rng = np.random.default_rng(12)
    P = _ln_rows(rng, 30000, 768)
    Q = _ln_rows(np.random.default_rng(13), 100, 768)
    idx = _index(P)
    D, I = idx.search_device(torch.from_numpy(Q).cuda(), 100, exact=True)
    Do, Io = flat_ip_oracle.search(P, Q, 100)
    assert (I.cpu().numpy() == Io).all() and (D.cpu().numpy() == Do).all()


def test_sharded_equals_global_on_one_gpu():
    """SURVEY.md §8(e) on one device: 4 row shards (i % 4), per-shard top-k with offsets, host merge."""
    from ance_b200.search import merge_topk_host
    rng = np.random.default_rng(14)
    P = _ln_rows(rng, 40001, 768)
    Q = _ln_rows(np.random.default_rng(15), 128, 768)
    W, k = 4, 100
    order = np.concatenate([np.arange(r, P.shape[0], W) for r in range(W)])
    Pm = P[order]
    Dg, Ig = flat_ip_oracle.search(Pm, Q, k)
    Ds, Is, off = [], [], 0
    qd = torch.from_numpy(Q).cuda()
    for r in range(W):
        n = len(range(r, P.shape[0], W))
        D, I = _index(Pm[off:off + n]).search_device(qd, k, row_offset=off)
        Ds.append(D.cpu().numpy())
        Is.append(I.cpu().numpy())
        off += n
    Dm, Im = merge_topk_host(Ds, Is, k)
    assert (Im == Ig).all() and (Dm == Dg).all()


def test_full_size_properties():
    """BASELINE config 2 size (8,841,823 x 768): properties that do not need a full-size CPU oracle."""
    from ance_b200.search import IndexFlatIP
    dev = torch.device("cuda:0")
    N, d, nq, k = 8841823, 768, 1024, 200
    idx = IndexFlatIP(d, capacity=N)
    g = torch.Generator(device=dev).manual_seed(1234)
    cent = torch.randn(1024, d, device=dev, generator=g)
    probe_rows = torch.randint(0, N, (nq,), generator=torch.Generator().manual_seed(3))
    keep = {}
    for s in range(0, N, 1 << 20):
        e = min(N, s + (1 << 20))
        x = 0.5 * torch.randn(e - s, d, device=dev, generator=g) + 0.5 * cent[torch.randint(0, 1024, (e - s,), device=dev, generator=g)]
        x = (x - x.mean(1, keepdim=True)) / x.std(1, keepdim=True, unbiased=False)
        idx.add(x)
        m = (probe_rows >= s) & (probe_rows < e)
        for qi in torch.nonzero(m).flatten().tolist():
            keep[qi] = x[probe_rows[qi] - s].clone()
    assert idx.ntotal == N
    Q = torch.stack([keep[i] for i in range(nq)]) * 1.5  # query i is a scaled copy of row probe_rows[i]
    D, I = idx.search_device(Q.contiguous(), k)
    torch.cuda.synchronize()
    # (1) the planted row is the top hit (Cauchy-Schwarz: all rows have the same norm)
    assert (I[:, 0].cpu() == probe_rows).all()
    # (2) sorted descending, labels in range and unique per query
    assert (D[:, 1:] <= D[:, :-1]).all() and (I >= 0).all() and (I < N).all()
    assert all(len(set(r)) == k for r in I[:64].cpu().tolist())
    # (3) identical to the exact brute-force kernel on a slice of the queries
    De, Ie = idx.search_device(Q[:32].contiguous(), k, exact=True)
    assert (I[:32] == Ie).all() and (D[:32] == De).all()
    assert idx.stats()["nq"] == nq


def test_tier2_threshold_pass_is_cheap_and_exact():
    """VERDICT r1 weak 3 (certification cliff): force ~all queries to fail the tier-1 certificate (bf16 operands, k' barely
    above k) and check that (i) tier 2 — the same coarse kernel restarted from each query's own threshold — certifies
    them all, (ii) the answer is the exact one, (iii) the whole search stays within 3x of a search whose certificates
    all pass at tier 1 (it was 25x with the fp64 brute force as the only fallback)."""
    rng = np.random.default_rng(31)
    N, nq, k = 1_000_000, 2048, 200
    P = np.concatenate([_ln_rows(np.random.default_rng(100 + i), 250_000, 768) for i in range(4)])
    Q = _ln_rows(np.random.default_rng(32), nq, 768)
    qd = torch.from_numpy(Q).cuda()

    def timed(idx):
        idx.search_device(qd, k)      # warm-up (workspace allocation)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        D, I = idx.search_device(qd, k)
        e1.record()
        torch.cuda.synchronize()
        return D.cpu().numpy(), I.cpu().numpy(), e0.elapsed_time(e1), idx.stats()

    # n_splits = 1 in both runs: with row-range splits every split keeps its own k' best rows and the certificate passes
    # trivially, which is not the regime (503k queries, one sweep per query tile) this test is about
    good = _index(P, "bf16", n_splits=1)          # default k' (432 for k = 200 with bf16): certifies at tier 1
    Dg, Ig, ms_good, st_good = timed(good)
    assert st_good["n_tier2"] == 0 and st_good["n_uncertified"] == 0
    del good
    tight = _index(P, "bf16", kprime=224, n_splits=1)   # eps ~ 3 needs ~300 rows above the cut: tier 1 must fail broadly
    Dt, It, ms_tight, st_tight = timed(tight)
    assert st_tight["n_tier2"] >= 0.3 * nq, st_tight
    assert st_tight["n_uncertified"] == 0, st_tight      # tier 2 certified every one of them: no brute force
    assert (It == Ig).all() and (Dt == Dg).all()
    Do, Io = flat_ip_oracle.search(P, Q[:32], k)
    assert (Ig[:32] == Io).all() and (Dg[:32] == Do).all()
    print(f"tier-1-only {ms_good:.1f} ms, {st_tight['n_tier2']}/{nq} through tier 2: {ms_tight:.1f} ms")
    assert ms_tight <= 3.0 * ms_good, (ms_tight, ms_good)


def test_tensor_core_accumulation_error_is_inside_the_certificate_bound(lib):
    """The certificate charges d * 2^-22 * |q^| |p^| for the tensor core's fp32 accumulation (search.cu,
    coarse_rescore_pass).  Measure the real thing: tensor-core scores of 16-bit operands against the fp64 dot product of
    the SAME rounded operands."""
    import ctypes as C
    torch.manual_seed(5)
    M, N, K = 256, 8192, 768
    worst = 0.0
    for fmt, dt in ((0, torch.float16), (1, torch.bfloat16)):
        A = torch.randn(M, K, device="cuda").to(dt)
        B = (torch.randn(N, K, device="cuda") * torch.rand(N, 1, device="cuda") * 4).to(dt)   # mixed row norms
        C32 = torch.full((M, N), float("nan"), device="cuda")
        rc = lib.ance_dbg_gemm(A.data_ptr(), B.data_ptr(), M, N, K, fmt, 2, None, None, 0, None, C32.data_ptr(),
                               C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, lib.ance_last_error()
        torch.cuda.synchronize()
        ref = A.double() @ B.double().t()
        scale = A.double().norm(dim=1)[:, None] * B.double().norm(dim=1)[None, :]
        rel = ((C32.double() - ref).abs() / scale).max().item()
        worst = max(worst, rel)
        assert rel <= K * 2.0 ** -22, (fmt, rel)
    print(f"max accumulation error / (|q||p|) = {worst:.3e}; bound {K * 2.0 ** -22:.3e} ({K * 2.0 ** -22 / worst:.0f}x)")


def test_non_finite_operands_are_refused_and_auto_falls_back_to_bf16():
    from ance_b200._lib import AnceError
    from ance_b200 import _lib
    rng = np.random.default_rng(41)
    P = _ln_rows(rng, 20000, 768)
    Q = _ln_rows(np.random.default_rng(42), 40, 768)
    # (i) a row outside the fp16 range: fp16 refuses, bf16 and auto answer exactly
    Pbig = P.copy()
    Pbig[777] *= 1.0e4                      # |x| up to ~4e4 * ... > 65504 for some component
    Pbig[777, 0] = 1.0e5
    Do, Io = flat_ip_oracle.search_bruteforce(Pbig, Q, 10)   # (the blocked oracle's fp32 noise bound scales with max |p|)
    with pytest.raises(AnceError, match="fp16"):
        _index(Pbig, "fp16").search(Q, 10)
    for operand in ("bf16", "auto"):
        idx = _index(Pbig, operand)
        D, I = idx.search(Q, 10)
        assert (I == Io).all() and (D == Do).all()
        assert idx.operand == _lib.ANCE_FMT_BF16
    # (ii) inf / NaN anywhere: every format refuses (the reference's faiss would return garbage silently)
    Pnan = P.copy()
    Pnan[5, 5] = np.nan
    for operand in ("auto", "bf16"):
        with pytest.raises(AnceError, match="non-finite"):
            _index(Pnan, operand).search(Q, 10)
    Qinf = Q.copy()
    Qinf[3, 0] = np.inf
    idx = _index(P)
    with pytest.raises(AnceError, match="query"):
        idx.search(Qinf, 10)
    D, I = idx.search(Q, 10)               # the query flag is per search: the index stays usable
    Do, Io = flat_ip_oracle.search(P, Q, 10)
    assert (I == Io).all() and (D == Do).all()


def test_index_over_caller_storage_adds_in_place():
    """ance_index_create_over: rows written by their producer straight into the index's storage are added without a
    copy (the refresher's memory path: one fp32 copy of the corpus)."""
    from ance_b200.search import IndexFlatIP
    rng = np.random.default_rng(51)
    P = _ln_rows(rng, 30000, 768)
    Q = _ln_rows(np.random.default_rng(52), 64, 768)
    store = torch.empty((30000, 768), dtype=torch.float32, device="cuda")
    idx = IndexFlatIP(768, storage=store)
    for s in range(0, 30000, 7000):                    # "encode" a slice into the storage, then add that very slice
        store[s:s + 7000].copy_(torch.from_numpy(P[s:s + 7000]))
        idx.add(store[s:s + 7000])
    assert idx.ntotal == 30000
    D, I = idx.search(Q, 100)
    Do, Io = flat_ip_oracle.search(P, Q, 100)
    assert (I == Io).all() and (D == Do).all()
    with pytest.raises(ValueError):
        IndexFlatIP(768, storage=torch.empty((10, 64), device="cuda"))


def test_centering_certifies_concentrated_embeddings():
    """Embeddings that share a large common component (anisotropic BERT-style outputs; an untrained / collapsed encoder —
    what the seeded-random checkpoints of this repo's own full-refresh runs produce): the score differences that decide the
    ranking are tiny next to the scores.  The index centres its rows before rounding them to 16 bits, so the certificate's
    error bound scales with the spread, not with the common component: everything certifies at tier 1; without the centring
    the same data falls through to the brute force."""
    rng = np.random.default_rng(61)
    n, nq, k = 200_000, 256, 100
    common = _ln_rows(rng, 1, 768, clustered=False)
    P = (common + 0.1 * rng.standard_normal((n, 768))).astype(np.float32)
    Q = (common + 0.1 * np.random.default_rng(62).standard_normal((nq, 768))).astype(np.float32)
    idx = _index(P, "fp16", n_splits=1)
    D, I = idx.search(Q, k)
    st = idx.stats()
    Do, Io = flat_ip_oracle.search(P, Q[:48], k)
    assert (I[:48] == Io).all() and (D[:48] == Do).all()
    assert st["n_tier2"] == 0 and st["n_uncertified"] == 0 and st["max_eps"] < 0.1, st
    raw = _index(P, "fp16", n_splits=1, center=0)
    D2, I2 = raw.search(Q, k)
    st2 = raw.stats()
    assert (I2 == I).all() and (D2 == D).all()                 # still exact, the expensive way
    assert st2["max_eps"] > 5 * st["max_eps"] and st2["n_tier2"] > nq // 2, (st, st2)
