"""Flat-IP search past its internal boundaries, at the query counts the refresh runs: large-k query blocks, brute-force
query batches, tier 2 and tier 3 inside later blocks, the host index's batch loop, workspace reuse, and the range checks
in a later block.  Every assertion is bit-exact (int64 labels, fp32 scores as bit patterns).

Two kinds of reference:
* an fp64 one.  Tie queries (near a group of identical rows) go to the CPU oracle's brute force.  Every other query goes
  to `_reference`: candidates from an fp64 GEMM, then each candidate's score summed in fp64 in the order of the kernel that
  produces it (`_order_sum`), rounded once to fp32, sorted by (score desc, row asc).  At tens of millions of compared
  scores, an fp64 sum in another order (BLAS) would round to a different fp32 value now and then.  `_reference` is held to
  `flat_ip_oracle.search` on a sample of queries.
* composition: the answer does not depend on how queries are grouped, so a call that crosses a boundary must be
  `torch.equal` to smaller calls that stay below it.

Each test also proves that its boundary was crossed: `ance_profile_read` counts one "exact" span per brute-force batch and
one "coarse_search" / "rescore" span per coarse pass, and the expected counts are derived below from search.cu's
constants.  If a constant changes, the count assertions fail instead of silently no longer crossing."""
import functools

import numpy as np
import pytest
import torch

from oracle import flat_ip_oracle

pytestmark = pytest.mark.gpu

DIM = 768
# ance_b200/csrc/search.cu
K_EXACT_BATCH = 1024                 # kExactBatch: queries per brute-force pass
K_EXACT_KEYS_BYTES = 512 << 20       # kExactKeysBytes: chunk keys per pass for k > 512
K_EXQB = 4                           # kExQB: queries per exact_chunk_kernel group
K_EX_GY_MAX = 128                    # exact_chunk_kernel's grid y cap: groups beyond it loop in the block
K_WIDE_QBLOCK = 16384                # kWideQBlock: query block of the large-k path
K_HOST_STAGE_BYTES = 512 << 20       # kHostStageBytes: a host index's brute-force slab
WORKSPACE_BOUND = 2.2e9              # include/ance_b200.h: large-k workspace "about 2.2 GB" whatever nq is


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _n_chunks(n):
    return max(1, min(2 * _sms(), -(-n // 4096)))


def _exact_batch(n_chunks, k, host=False):
    """run_exact / run_exact_host: queries per brute-force batch (a host index keeps one more key slot per query)."""
    b = K_EXACT_BATCH
    if k > 512:
        per_query = (n_chunks + (1 if host else 0)) * k * 8
        b = min(b, max(K_EXQB, K_EXACT_KEYS_BYTES // per_query // K_EXQB * K_EXQB))
    return b


def _split(nq, b):
    return [min(b, nq - s) for s in range(0, nq, b)]


def _blocks(nq):
    """ance_index_search, k > 512: equal blocks of at most kWideQBlock, rounded up to the 256-query tile."""
    n_blocks = -(-nq // K_WIDE_QBLOCK)
    return _split(nq, min(K_WIDE_QBLOCK, -(-(-(-nq // n_blocks)) // 256) * 256))


def _idx(P, operand="fp16", rows="device"):
    from ance_b200.search import IndexFlatIP
    idx = IndexFlatIP(DIM, capacity=P.shape[0], operand=operand, rows=rows)
    idx.add(P)
    return idx


def _profiled(fn):
    from ance_b200 import _lib
    _lib.profile_enable(True)
    _lib.profile_read(reset=True)
    try:
        out = fn()
    finally:
        prof = _lib.profile_read(reset=True)
        _lib.profile_enable(False)
    return out, {c: prof[c][1] for c in ("coarse_search", "rescore", "exact")}


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else x


def _same(D, I, Do, Io, what=""):
    D, I, Do, Io = _np(D), _np(I), _np(Do), _np(Io)
    bad = (I != Io).any(1) | (D.view(np.uint32) != Do.view(np.uint32)).any(1)
    assert not bad.any(), f"{what}: {bad.sum()} of {len(bad)} queries differ, first {np.flatnonzero(bad)[:8]}"


# ------------------------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------------------------
def _order_sum(prod, order):
    """Sum fp64 products over the last axis (d = 768) in a kernel's order.  "rescore": warp_dots_f64, lane l adds
    elements j·128 + 4l + t for j = 0..5, t = 0..3.  "exact": exact_chunk_kernel, lane l adds elements l + 32m.  Then
    both kernels combine the lanes with the xor-shuffle tree 16, 8, 4, 2, 1.  fp32 × fp32 is exact in fp64, so each fma
    is one fp64 add."""
    if order == "rescore":
        x = prod.unflatten(-1, (6, 32, 4))
        terms = [x[..., j, :, t] for j in range(6) for t in range(4)]
    else:
        x = prod.unflatten(-1, (24, 32))
        terms = [x[..., m, :] for m in range(24)]
    acc = terms[0]
    for t in terms[1:]:
        acc = acc + t
    while acc.shape[-1] > 1:
        h = acc.shape[-1] // 2
        acc = acc[..., :h] + acc[..., h:]
    return acc[..., 0]


def _reference(P, Q, k, order, slack=64, qb=64):
    """(D, I) on the device for queries without exact ties (see the module docstring)."""
    Pd = P.double()
    pmax = Pd.norm(dim=1).max()
    Ds, Is = [], []
    for q0 in range(0, Q.shape[0], qb):
        q = Q[q0:q0 + qb].double()
        c_s, c_i = (q @ Pd.T).topk(min(P.shape[0], k + slack), dim=1)
        s = _order_sum(q[:, None, :] * Pd[c_i], order)
        c_i, perm = c_i.sort(dim=1)                          # rows ascending, so that the stable sort below ...
        s = s.gather(1, perm)
        s32, o = s.float().sort(dim=1, descending=True, stable=True)   # ... breaks score ties by the lower row
        kth = s.gather(1, o[:, k - 1:k])[:, 0]
        # a non-candidate scores at most c_s[-1] + err: it must round strictly below the k-th score
        err = DIM * 2.0 ** -52 * q.norm(dim=1) * pmax
        assert (kth - c_s[:, -1] > 2 * err + kth.abs() * 2.0 ** -22).all(), "reference slack too small"
        Ds.append(s32[:, :k])
        Is.append(c_i.gather(1, o[:, :k]))
    return torch.cat(Ds), torch.cat(Is)


def _bruteforce(Pn, Qn, k):
    """flat_ip_oracle.search_bruteforce, 64 queries at a time."""
    parts = [flat_ip_oracle.search_bruteforce(Pn, Qn[s:s + 64], k) for s in range(0, Qn.shape[0], 64)]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


# ------------------------------------------------------------------------------------------------------------------
# corpora, generated on the device from seeds
# ------------------------------------------------------------------------------------------------------------------
def _rows(n, seed, clustered=True):
    """LayerNorm-like rows, clustered around 64 shared centres (as test_full_size_properties)."""
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(n, DIM, device=dev, generator=g)
    if clustered:
        cent = torch.randn(64, DIM, device=dev, generator=torch.Generator(device=dev).manual_seed(7))
        x = 0.5 * x + 0.5 * cent[torch.randint(0, 64, (n,), device=dev, generator=g)]
    return ((x - x.mean(1, keepdim=True)) / x.std(1, keepdim=True, unbiased=False)).contiguous()


def _tie_world(n, nq, groups, near, seed, spread=()):
    """n rows, `groups[g]` of them set to one shared vector v_g (plus 1e-4 noise per row for the groups listed in
    `spread`: rows the 16-bit pass cannot tell apart, but with distinct exact scores, so that an answer tiers 1 and 2
    leave uncertified is also wrong).  Query positions `near[g]` are v_g + 5 % noise: their top k are rows of group g.
    Every other query is pushed away from every group (score about -0.5 · 768 with each), so no group reaches its top
    2048."""
    P = _rows(n, seed)
    v = _rows(len(groups), seed + 1, clustered=False)
    for g, rows in enumerate(groups):
        rows = torch.as_tensor(rows, device=P.device)
        P[rows] = v[g] + (1e-4 * _rows(len(rows), seed + 4 + g) if g in spread else 0)
    Q = _rows(nq, seed + 2) - 0.5 * v.sum(0)
    noise = _rows(nq, seed + 3)
    for g, pos in enumerate(near):
        pos = torch.as_tensor(pos, device=P.device)
        Q[pos] = v[g] + 0.05 * noise[pos]
    return P.contiguous(), Q.contiguous(), v


# Case 1: 400,000 ordinary rows, 2,500 queries.
N1 = 400_000


@functools.lru_cache(maxsize=None)
def _world1():
    P, Q = _rows(N1, 11), _rows(2500, 12)
    return P, Q, P.cpu().numpy(), Q.cpu().numpy()


@functools.lru_cache(maxsize=None)
def _index1():
    return _idx(_world1()[0])


@functools.lru_cache(maxsize=None)
def _exact1(k, nq):
    P, Q, *_ = _world1()
    return _profiled(lambda: _index1().search_device(Q[:nq], k, exact=True))


# Case 2: 300,000 rows, 16,384 of them near-identical (interleaved); 2,200 queries, those at odd positions near them.
N2 = 300_000
TIE2 = np.arange(0, 32768, 2)
NEAR2 = np.arange(1, 2200, 2)


@functools.lru_cache(maxsize=None)
def _world2():
    P, Q, _ = _tie_world(N2, 2200, [TIE2], [NEAR2], 21, spread=(0,))
    return P, Q, P.cpu().numpy(), Q.cpu().numpy()


# Case 3: 40,000 rows: group A, 16,384 identical rows interleaved (more than tier 2's 8,160: tier 3); group B, 3,000
# identical rows in one range (above k' = 1440 within a split, below 8,160: tier 2 only).  40,000 queries: block 0 of
# every call ordinary; near-A / near-B queries at non-contiguous positions from 13,568 on, including the last query of
# 16,385 / 18,944 / 40,000 and both sides of the 40,000-query call's second block boundary.
N3 = 40_000
A3 = np.arange(0, 32768, 2)
B3 = np.arange(34000, 37000)
NEAR_A3 = np.array(sorted(set(range(13568, 40000, 194)) | {16384, 27135}))
NEAR_B3 = np.array(sorted((set(range(13665, 40000, 194)) | {18943, 27136, 39999}) - set(NEAR_A3.tolist())))
SPECIAL3 = np.union1d(NEAR_A3, NEAR_B3)
ORD3 = np.setdiff1d(np.arange(40000), SPECIAL3)


@functools.lru_cache(maxsize=None)
def _world3():
    P, Q, _ = _tie_world(N3, 40000, [A3, B3], [NEAR_A3, NEAR_B3], 31)
    return P, Q, P.cpu().numpy(), Q.cpu().numpy()


@functools.lru_cache(maxsize=None)
def _ref3():
    """The answer at k = 2048 for all 40,000 queries (its first 1000 columns are the answer at k = 1000)."""
    P, Q, Pn, Qn = _world3()
    k = 2048
    D = torch.empty((40000, k), dtype=torch.float32, device="cuda")
    I = torch.empty((40000, k), dtype=torch.int64, device="cuda")
    o = torch.as_tensor(ORD3, device="cuda")
    D[o], I[o] = _reference(P, Q[o], k, "rescore")
    Ds, Is = _bruteforce(Pn, Qn[SPECIAL3], k)
    s = torch.as_tensor(SPECIAL3, device="cuda")
    D[s], I[s] = torch.from_numpy(Ds).cuda(), torch.from_numpy(Is).cuda()
    return D, I


def _in(pos, lo, hi):
    return int(((pos >= lo) & (pos < hi)).sum())


# ------------------------------------------------------------------------------------------------------------------
# boundaries the tests below rely on, with the numbers of a 132-SM H100 at d = 768
# ------------------------------------------------------------------------------------------------------------------
def test_boundary_numbers():
    assert _blocks(16385) == [8448, 7937]
    assert _blocks(18944) == [9472, 9472]
    assert _blocks(40000) == [13568, 13568, 12864]
    assert _blocks(16384) == [16384]
    assert _n_chunks(N1) == 98 and _n_chunks(N2) == 74 and _n_chunks(N3) == 10
    assert [_exact_batch(98, k) for k in (100, 1000, 2048)] == [1024, 684, 332]
    assert _exact_batch(74, 2048) == 440 and _exact_batch(74, 50) == 1024
    slab = K_HOST_STAGE_BYTES // (DIM * 4)
    assert slab == 174762 and -(-N1 // slab) == 3 and _n_chunks(slab) == 43 and _exact_batch(43, 100, host=True) == 1024
    if _sms() == 132:
        assert 4 * _sms() == 528


# ------------------------------------------------------------------------------------------------------------------
# 1. brute-force batches, device index
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,nq,batches", [(100, 2500, [1024, 1024, 452]), (1000, 1500, [684, 684, 132]),
                                          (2048, 700, [332, 332, 36])])
def test_exact_batches_device(k, nq, batches):
    P, Q, Pn, Qn = _world1()
    b = _exact_batch(_n_chunks(N1), k)
    assert _split(nq, b) == batches
    if k == 100:   # a block loops over a second group of 4 queries, a merge block over a second query
        assert batches[0] > K_EXQB * K_EX_GY_MAX and batches[0] > 4 * _sms()
    (D, I), spans = _exact1(k, nq)
    assert spans["exact"] == len(batches), spans
    # composition: 4-query calls (one group, one query per merge block) give the same tensors
    parts = [_index1().search_device(Q[s:s + 4], k, exact=True) for s in range(0, nq, 4)]
    assert torch.equal(D, torch.cat([p[0] for p in parts])) and torch.equal(I, torch.cat([p[1] for p in parts]))
    # every query against the fp64 reference in exact_chunk_kernel's order
    _same(D, I, *_reference(P, Q[:nq], k, "exact"), what="reference")
    # the CPU oracle on the first and last query of every batch and 32 more
    edges = {e for s in range(0, nq, b) for e in (s, min(nq, s + b) - 1)}
    rng = np.random.default_rng(k)
    sample = np.array(sorted(edges | set(rng.choice(nq, 32, replace=False).tolist())))
    _same(D[sample], I[sample], *_bruteforce(Pn, Qn[sample], k), what="oracle")


# ------------------------------------------------------------------------------------------------------------------
# 2. tier 3 with many flagged queries
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [50, 2048])
def test_tier3_many_flagged(k):
    P, Q, Pn, Qn = _world2()
    idx = _idx(P)
    (D, I), spans = _profiled(lambda: idx.search_device(Q, k))
    st = idx.stats()
    b = _exact_batch(_n_chunks(N2), k)
    assert b == (440 if k == 2048 else 1024)
    assert st["n_uncertified"] == len(NEAR2), st
    assert spans["exact"] == len(_split(len(NEAR2), b)) >= 2, spans   # k = 50: 1024 + 76; k = 2048: 440 + 440 + 220
    assert spans["coarse_search"] == spans["rescore"] == 2, spans      # tier 1 and tier 2, one block
    near = torch.as_tensor(NEAR2, device="cuda")
    De, Ie = idx.search_device(Q[near], k, exact=True)
    assert torch.equal(D[near], De) and torch.equal(I[near], Ie)
    # every near query against the reference in exact_chunk_kernel's order (its k-th row has thousands of neighbours
    # within 1e-3: a wide candidate slack)
    assert np.isin(I[near].cpu().numpy(), TIE2).all()
    _same(D[near], I[near], *_reference(P, Q[near], k, "exact", slack=2048), what="near")
    ordinary = torch.as_tensor(np.setdiff1d(np.arange(2200), NEAR2), device="cuda")
    _same(D[ordinary], I[ordinary], *_reference(P, Q[ordinary], k, "rescore"), what="ordinary")
    # the CPU oracle on the first and last near query, the near queries on both sides of every batch boundary of their
    # sorted list, and ordinary ones
    cut = {NEAR2[0], NEAR2[-1]} | {NEAR2[i] for s in range(b, len(NEAR2), b) for i in (s - 1, s)}
    rng = np.random.default_rng(k)
    sample = np.array(sorted(cut | set(rng.choice(2200, 64 - len(cut), replace=False).tolist())))
    _same(D[sample], I[sample], *_bruteforce(Pn, Qn[sample], k), what="oracle")


# ------------------------------------------------------------------------------------------------------------------
# 3. large-k query blocks
# ------------------------------------------------------------------------------------------------------------------
def test_reference_equals_oracle():
    """`_reference` against the CPU oracle on ordinary queries, including both sides of every block boundary."""
    P, Q, Pn, Qn = _world3()
    edges = [0, 8447, 8448, 9471, 9472, 13567, 16383, 18942, 27134, 27137, 39998]
    sample = np.union1d(np.intersect1d(edges, ORD3), np.random.default_rng(3).choice(ORD3, 48, replace=False))
    Do, Io = _ref3()
    _same(Do[sample], Io[sample], *flat_ip_oracle.search(Pn, Qn[sample], 2048), what="reference")


@pytest.mark.parametrize("nq,k,operand", [(16385, 1000, "fp16"), (18944, 1000, "fp16"), (40000, 1000, "fp16"),
                                          (16385, 2048, "bf16")])
def test_large_k_query_blocks(nq, k, operand):
    P, Q, *_ = _world3()
    idx = _idx(P, operand)
    (D, I), spans = _profiled(lambda: idx.search_device(Q[:nq], k))
    st = idx.stats()
    Do, Io = _ref3()
    _same(D, I, Do[:nq, :k], Io[:nq, :k], what="reference")
    # each block equals that block searched alone, and the call's statistics combine the blocks'
    blocks = _blocks(nq)
    assert len(blocks) >= 2
    alone, b0 = [], 0
    for nb in blocks:
        (Db, Ib), sp = _profiled(lambda: idx.search_device(Q[b0:b0 + nb].contiguous(), k))
        assert torch.equal(D[b0:b0 + nb], Db) and torch.equal(I[b0:b0 + nb], Ib), (b0, nb)
        sb = idx.stats()
        n_a, n_b = _in(NEAR_A3, b0, b0 + nb), _in(NEAR_B3, b0, b0 + nb)
        assert sb["n_uncertified"] == n_a, (b0, sb)       # near A: tier 3; everything else certified
        if operand == "fp16":
            assert sb["n_tier2"] >= n_a + n_b, (b0, sb)   # near B: through tier 2
        if b0 > 0:
            assert n_a > 0 and n_b > 0                    # tier 2 and tier 3 inside a later block
        alone.append((sb, sp))
        b0 += nb
    want = {"nq": nq, "kprime": alone[0][0]["kprime"]}
    for f in ("n_tier2", "n_uncertified", "n_candidates"):
        want[f] = sum(s[f] for s, _ in alone)
    for f in ("n_splits", "max_eps"):
        want[f] = max(s[f] for s, _ in alone)
    assert st == want, (st, want)
    # profile: one tier-1 pass per block, one tier-2 pass per block that flagged, one exact span per tier-3 batch
    b = _exact_batch(_n_chunks(N3), k)
    tiers = sum(1 + (s["n_tier2"] > 0) for s, _ in alone)
    exact = sum(len(_split(s["n_uncertified"], b)) for s, _ in alone)
    assert spans == {"coarse_search": tiers, "rescore": tiers, "exact": exact}, spans
    assert spans == {c: sum(sp[c] for _, sp in alone) for c in spans}
    assert tiers >= len(blocks) + len(blocks) - 1 and exact >= len(blocks) - 1


N3B = 40_000
T2B = np.arange(20000, 20600)          # 600 identical rows in one range: tier 2 (above k' = 288 within a split)
T3B = np.arange(0, 16384, 2)           # 8,192 near-identical rows, interleaved: more than tier 2's 2,016 (k' = 992)
NEAR_T3B = np.arange(3, 18944, 17)[:1100]
NEAR_T2B = np.setdiff1d(np.arange(5, 18944, 61), NEAR_T3B)[:300]


@functools.lru_cache(maxsize=None)
def _world3b():
    P, Q, _ = _tie_world(N3B, 18944, [T2B, T3B], [NEAR_T2B, NEAR_T3B], 41, spread=(1,))
    return P, Q, P.cpu().numpy(), Q.cpu().numpy()


def test_small_k_driver_call_tier3_two_batches():
    """The driver's real call: one 18,944-query block at k = 200 (no blocking below k = 512), with more than 1,024
    queries left to the brute force, so that tier 3 runs two batches."""
    P, Q, Pn, Qn = _world3b()
    k = 200
    idx = _idx(P)
    (D, I), spans = _profiled(lambda: idx.search_device(Q, k))
    st = idx.stats()
    b = _exact_batch(_n_chunks(N3B), k)
    assert len(NEAR_T3B) == 1100 > b == 1024
    assert st["n_uncertified"] == len(NEAR_T3B) and st["n_tier2"] >= len(NEAR_T3B) + len(NEAR_T2B), st
    assert spans == {"coarse_search": 2, "rescore": 2, "exact": 2}, spans
    t3 = torch.as_tensor(NEAR_T3B, device="cuda")
    De, Ie = idx.search_device(Q[t3], k, exact=True)
    assert torch.equal(D[t3], De) and torch.equal(I[t3], Ie)
    assert np.isin(I[t3].cpu().numpy(), T3B).all()
    _same(D[t3], I[t3], *_reference(P, Q[t3], k, "exact", slack=2048), what="tier 3")
    ordinary = np.setdiff1d(np.arange(18944), np.union1d(NEAR_T3B, NEAR_T2B))
    o = torch.as_tensor(ordinary, device="cuda")
    _same(D[o], I[o], *_reference(P, Q[o], k, "rescore"), what="ordinary")
    _same(D[NEAR_T2B], I[NEAR_T2B], *_bruteforce(Pn, Qn[NEAR_T2B], k), what="tier 2")
    sample = np.array(sorted({NEAR_T3B[0], NEAR_T3B[b - 1], NEAR_T3B[b], NEAR_T3B[-1]}
                             | set(np.random.default_rng(5).choice(NEAR_T3B, 28, replace=False).tolist())))
    _same(D[sample], I[sample], *_bruteforce(Pn, Qn[sample], k), what="tier 3 oracle")


# ------------------------------------------------------------------------------------------------------------------
# 4. host index
# ------------------------------------------------------------------------------------------------------------------
def test_host_index_blocks_equal_device():
    P, Q, *_ = _world3()
    q, k = Q[:18944], 1000
    h, d = _idx(P, rows="host"), _idx(P)
    (Dh, Ih), sph = _profiled(lambda: h.search_device(q, k))
    (Dd, Id), spd = _profiled(lambda: d.search_device(q, k))
    assert torch.equal(Dh, Dd) and torch.equal(Ih, Id)
    assert h.stats() == d.stats() and sph == spd and spd["coarse_search"] >= 3, (h.stats(), d.stats(), sph, spd)
    assert h.last_fetched() > 0 and d.last_fetched() == 0


def test_host_index_exact_batches_over_slabs():
    """400,000 host rows are three brute-force slabs; 1,100 queries are two batches.  The running best-k slot of every
    query is cleared per batch: a stale slot would leak the first batch's rows into the second's answers."""
    P, Q, *_ = _world1()
    nq, k = 1100, 100
    slab = K_HOST_STAGE_BYTES // (DIM * 4)
    assert -(-N1 // slab) == 3
    assert _split(nq, _exact_batch(_n_chunks(slab), k, host=True)) == [1024, 76]
    h = _idx(P, rows="host")
    (D, I), spans = _profiled(lambda: h.search_device(Q[:nq], k, exact=True))
    assert spans["exact"] == 2, spans
    (Dd, Id), _ = _exact1(k, 2500)
    assert torch.equal(D, Dd[:nq]) and torch.equal(I, Id[:nq])


# ------------------------------------------------------------------------------------------------------------------
# 5. workspace reuse
# ------------------------------------------------------------------------------------------------------------------
def _own_bytes(n):
    """memory()["device"] of a device index that has not searched: fp32 rows, 16-bit operands, pstats, pace, counters,
    mu, colsum (ance_index_memory)."""
    return 6 * n * DIM + 2 * 4 + 256 * 4 + 8 * 4 + DIM * 4 + DIM * 8


def test_workspace_reuse_across_shapes():
    P, Q, *_ = _world3()
    idx = _idx(P)
    assert idx.memory()["device"] == _own_bytes(N3)
    for nq, k, exact in ((300, 200, False), (40000, 1000, False), (7, 2048, False), (2500, 100, True),
                         (18944, 200, False), (1, 1, False), (16385, 2048, False)):
        D, I = idx.search_device(Q[:nq], k, exact=exact)
        Df, If = _idx(P).search_device(Q[:nq], k, exact=exact)
        assert torch.equal(D, Df) and torch.equal(I, If), (nq, k, exact)
    ws = idx.memory()["device"] - _own_bytes(N3)
    assert 0 < ws <= WORKSPACE_BOUND, ws
    # the large-k workspace does not grow with nq: a 40,000-query search needs no more than its three blocks searched
    # one after the other.  (Not "no more than any 16,384-query search": the row-range split count follows the block
    # size, and a 12,864-query block takes 5 ranges of k' candidates where 16,384 queries take one.)
    a, b = _idx(P), _idx(P)
    b0 = 0
    for nb in _blocks(40000):
        a.search_device(Q[b0:b0 + nb].contiguous(), 1000)
        b0 += nb
    b.search_device(Q[:40000], 1000)
    assert b.stats()["n_uncertified"] > 0 and b.stats()["n_splits"] > 1, b.stats()
    assert b.memory()["device"] <= a.memory()["device"], (a.memory(), b.memory())
    assert b.memory()["device"] - _own_bytes(N3) <= WORKSPACE_BOUND


# ------------------------------------------------------------------------------------------------------------------
# 6. range fallbacks in a later block
# ------------------------------------------------------------------------------------------------------------------
def test_range_fallbacks_in_last_block():
    from ance_b200 import _lib
    P, Q, Pn, Qn = _world3()
    nq, k = 16385, 1000
    last0 = nq - _blocks(nq)[-1]
    pos = int(ORD3[ORD3 < nq][-1])
    assert pos >= last0
    Do, Io = _ref3()
    # |x| > 65504 in the last block: "auto" re-rounds the index to bf16 and answers every query exactly
    Qb = Q[:nq].clone()
    Qb[pos] *= 3.0e4
    assert Qb[pos].abs().max() > 65504
    idx = _idx(P, "auto")
    D, I = idx.search_device(Qb, k)
    assert idx.operand == _lib.ANCE_FMT_BF16
    keep = np.setdiff1d(np.arange(nq), [pos])
    _same(D[keep], I[keep], Do[keep, :k], Io[keep, :k], what="others")
    _same(D[pos:pos + 1], I[pos:pos + 1], *_reference(P, Qb[pos:pos + 1], k, "rescore"), what="scaled query")
    _same(D[pos:pos + 1], I[pos:pos + 1], *flat_ip_oracle.search_bruteforce(Pn, Qb[pos:pos + 1].cpu().numpy(), k))
    # NaN in the last block: refused; the index stays usable
    Qn_ = Q[:nq].clone()
    Qn_[pos, 5] = float("nan")
    idx2 = _idx(P, "auto")
    with pytest.raises(_lib.AnceError, match="non-finite"):
        idx2.search_device(Qn_, k)
    D, I = idx2.search_device(Q[:nq], k)
    _same(D, I, Do[:nq, :k], Io[:nq, :k], what="after the refusal")
