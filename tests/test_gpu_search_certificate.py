"""The flat-IP search's exactness certificate, tested directly (references and bounds: tests/search_refs.py).

1. The certificate's inputs against fp64: the centre mu, the 16-bit operand rows, the residual norms and their maxima, the
   query norms, read from the index with ance_dbg_index_state.
2. The coarse pass's candidate contract (EpTopK): per (query, split), every row whose coarse score exceeds the exported
   threshold is a candidate, every candidate reaches it, and ties at it keep the lowest rows; coarse scores recomputed from
   the exported operands by the same tensor-core mainloop (ance_dbg_gemm).
3. Corpora whose rounding residuals are aligned with the query, so that tier 1's answer is wrong and only eps keeps the
   certificate from accepting it: tier 1 alone flags every wrong query, and the full search returns the oracle's answer.
"""
import functools

import numpy as np
import pytest
import torch

from ance_b200 import _lib
from oracle import flat_ip_oracle
from tests import search_refs as sr
from tests.test_gpu_search import _ln_rows

pytestmark = pytest.mark.gpu

F32_NEG_INF = float("-inf")


def _make(P, fmt, host=False, **params):
    from ance_b200.search import IndexFlatIP
    idx = IndexFlatIP(P.shape[1], capacity=P.shape[0], operand=fmt, rows="host" if host else "device")
    idx.add(P)
    for k, v in params.items():
        idx.set_param(k, v)
    return idx


def _state(idx, item, shape, dtype):
    out = torch.empty(shape, dtype=dtype)
    _lib.index_state(idx._h, item, out)
    return out.numpy()


def _pass(idx):
    return dict(zip(("nq", "n_splits", "out_cap", "kprime", "rows_per_split", "tier"), _state(idx, "pass", 6, torch.int32)))


def _ord(x: torch.Tensor) -> torch.Tensor:
    """The kernels' order-preserving key of fp32 values (f2ord), as int64 (-0 < +0, as in the coarse pass)."""
    u = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    return torch.where(u >= 0x80000000, u ^ 0xFFFFFFFF, u | 0x80000000)


# ---------------------------------------------------------------------------------------------------------------------
# 1. operands
# ---------------------------------------------------------------------------------------------------------------------
def _edge_rows(rng, n, d, fmt):
    P = _ln_rows(rng, n, d)
    big = 60000.0 if fmt == "fp16" else 1e15
    P[5] = np.where(rng.random(d) < 0.5, big, -big)      # fp16: components near +-65504
    P[6] = rng.standard_normal(d) * 1e-6                 # the fp16 subnormal range: large relative residual
    P[7] = 0.3                                           # a constant row
    P[8] = P[7] * -1
    return P


@pytest.mark.parametrize("host", [False, True])
@pytest.mark.parametrize("center", [0, 1])
@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
@pytest.mark.parametrize("d", [768, 256])
def test_operands_against_fp64(d, fmt, center, host):
    rng = np.random.default_rng(100 + d + center)
    n = 3000
    P = _edge_rows(rng, n, d, fmt)
    Q = _ln_rows(np.random.default_rng(7), 40, d)
    Q[3] *= 1e-6
    idx = _make(P, fmt, host, center=center)
    idx.search(Q, 10)
    centred = bool(_state(idx, "centred", 1, torch.int32)[0])
    assert centred == bool(center)
    mu = _state(idx, "mu", d, torch.float32) if centred else None
    if centred:
        ref = sr.mean_ref(P)
        assert (np.abs(mu.astype(np.float64) - ref) <= sr.ulp32(ref)).all()
    bits, hat, X = sr.operand_rows(P, mu, fmt)
    p16 = _state(idx, "p16", (n, d), torch.int16).view(np.uint16)
    assert (p16 == bits).all(), f"{(p16 != bits).any(1).sum()} rows differ"
    pn, pd, xn = sr.exact_norms(P, mu, hat)
    ps = _state(idx, "pstats", 2, torch.float32).astype(np.float64)
    assert ps[0] >= pn.max() and ps[0] <= sr.norm_upper(pn, xn, d, False).max()
    assert ps[1] >= pd.max() and ps[1] <= sr.norm_upper(pd, xn, d, centred).max()
    if host:
        nd = _state(idx, "ndelta", n, torch.float32)
        assert (nd >= pd).all() and (nd <= sr.norm_upper(pd, xn, d, centred)).all()
        assert np.float32(ps[1]) == nd.max()
    else:
        with pytest.raises(_lib.AnceError):
            _state(idx, "ndelta", n, torch.float32)
    qbits, qhat = sr.round16(Q, fmt)
    assert (_state(idx, "q16", Q.shape, torch.int16).view(np.uint16) == qbits).all()
    qn, qd, qx = sr.exact_norms(Q, None, qhat)
    qnk = _state(idx, "qn_hat", len(Q), torch.float32)
    qdk = _state(idx, "qn_delta", len(Q), torch.float32)
    assert (qnk >= qn).all() and (qnk <= sr.norm_upper(qn, qx, d, False)).all()
    assert (qdk >= qd).all() and (qdk <= sr.norm_upper(qd, qx, d, False)).all()


def test_centring_switches_on_at_256_rows():
    for n, want in ((255, 0), (256, 1)):
        idx = _make(_ln_rows(np.random.default_rng(n), n, 768), "fp16")
        idx.prepare()
        assert _state(idx, "centred", 1, torch.int32)[0] == want


def test_hook_refuses_what_the_last_search_does_not_hold():
    from ance_b200.search import IndexFlatIP
    P = _ln_rows(np.random.default_rng(3), 2000, 256)
    idx = IndexFlatIP(256, capacity=2008, operand="fp16")
    idx.add(P)
    with pytest.raises(_lib.AnceError):
        _state(idx, "q16", (4, 256), torch.int16)         # no search yet
    idx.search(P[:4], 10)
    _state(idx, "q16", (4, 256), torch.int16)
    with pytest.raises(_lib.AnceError):
        _state(idx, "q16", (5, 256), torch.int16)         # wrong size
    with pytest.raises(_lib.AnceError):
        _state(idx, "ndelta", 2000, torch.float32)        # a device index keeps none
    with pytest.raises(_lib.AnceError):
        _lib.check(_lib.load().ance_dbg_index_state(idx._h, 99, torch.empty(4).data_ptr(), 16, None))
    idx.add(P[:8])
    with pytest.raises(_lib.AnceError):
        _state(idx, "p16", (2008, 256), torch.int16)      # rows added since: the operands are stale


# ---------------------------------------------------------------------------------------------------------------------
# 2. the candidate contract
# ---------------------------------------------------------------------------------------------------------------------
def _coarse_scores(idx, nq, n, d, fmt, cg):
    """C = Q^ P^T from the exported operands, fp32, by the coarse pass's mainloop (BN 128, 4 stages, CG 1 or 2)."""
    q16 = torch.from_numpy(_state(idx, "q16", (nq, d), torch.int16)).cuda()
    npad = -(-n // 8) * 8
    p16 = torch.zeros((npad, d), dtype=torch.int16, device="cuda")
    p16[:n] = torch.from_numpy(_state(idx, "p16", (n, d), torch.int16)).cuda()
    C = torch.full((nq, npad), float("nan"), device="cuda")
    lib = _lib.load()
    _lib.check(lib.ance_dbg_gemm(q16.data_ptr(), p16.data_ptr(), nq, npad, d, 0 if fmt == "fp16" else 1,
                                 0 if cg == 1 else 2, None, None, 0, None, C.data_ptr(), _lib.current_stream()))
    torch.cuda.synchronize()
    return C[:, :n]


def _check_contract(idx, C, n, thr_floor=None):
    """Every (query, split) of the last coarse pass against the coarse scores C [nq, n] (CUDA).  thr_floor [nq]: tier 2's
    starting thresholds.  Returns the pass shape."""
    ps = _pass(idx)
    nq, ns, cap, kp, rps = ps["nq"], ps["n_splits"], ps["out_cap"], ps["kprime"], ps["rows_per_split"]
    assert C.shape[0] == nq and ns >= 1 and (ns - 1) * rps < n <= ns * rps
    ids = torch.from_numpy(_state(idx, "cand_id", (nq, ns, cap), torch.int32)).cuda().long()
    cnt = torch.from_numpy(_state(idx, "cand_cnt", (nq, ns), torch.int32)).cuda().long()
    thr = torch.from_numpy(_state(idx, "cand_thr", (nq, ns), torch.float32)).cuda()
    K = _ord(C)
    for s in range(ns):
        r0, r1 = s * rps, min(n, (s + 1) * rps)
        Ks, T, c = K[:, r0:r1], _ord(thr[:, s])[:, None], cnt[:, s]
        fin = torch.isfinite(thr[:, s])
        if thr_floor is None:
            # a threshold is one of the split's coarse scores: the two GEMM paths are bit-identical
            assert ((Ks == T).any(1) | ~fin).all(), f"split {s}: a threshold is not a coarse score of the split"
            assert (c[fin] == kp).all() and (c[~fin] == r1 - r0).all() and (thr[~fin, s] == F32_NEG_INF).all()
        else:
            assert (thr[:, s] >= thr_floor).all()
        col = torch.arange(cap, device="cuda")[None, :]
        valid = col < c[:, None]
        rid = ids[:, s]
        assert ((rid >= r0) & (rid < r1) | ~valid).all(), f"split {s}: candidate outside the split"
        mask = torch.zeros((nq, r1 - r0 + 1), dtype=torch.int32, device="cuda")
        mask.scatter_add_(1, torch.where(valid, rid - r0, r1 - r0), valid.int())
        assert (mask[:, :-1] <= 1).all(), f"split {s}: repeated candidate"
        m = mask[:, :-1].bool()
        assert (m.sum(1) == c).all()
        assert (m | (Ks <= T)).all(), f"split {s}: a row above the threshold is missing"
        if thr_floor is None:
            assert (~m | (Ks >= T)).all(), f"split {s}: a candidate below the threshold"
            eq = Ks == T
            kept_eq = (c - (Ks > T).sum(1))[:, None]
            assert ((m & eq) == (eq & (eq.cumsum(1) <= kept_eq))).all(), f"split {s}: ties not the lowest rows"
        else:
            F = _ord(thr_floor)[:, None]
            assert (~m | (Ks > F)).all()
            same = (thr[:, s] == thr_floor)[:, None]      # no compaction: exactly the rows above the floor
            assert (~same | (m == (Ks > F))).all()
    return ps


def _ties_corpus(n, d, q0, kp, seed, ascending=False):
    """Rows of _ln_rows; 48 copies of the row at rank ~k' - 20 of query q0 placed 3 apart in split 0 (exactly equal keys
    across the cut and across 32-entry chunks); ascending: rows sorted by their score against q0."""
    P = _ln_rows(np.random.default_rng(seed), n, d)
    s = P @ q0
    if ascending:
        return np.ascontiguousarray(P[np.argsort(s, kind="stable")])
    r = np.argsort(-s, kind="stable")[kp - 20]
    pos = 40 + 3 * np.arange(48)
    P[pos] = P[r]
    return P


CONTRACT_CASES = [
    # k, k', cta_group, n_splits, n rows      (k' <= 512: reservoirs of 1024; <= 992: 2048; larger: streaming 8192)
    (100, 160, 1, 1, 20000),
    (100, 160, 2, 16, 15 * 1280 + 100),      # 16 splits of 1280 rows, the last one 100 rows (< k')
    (200, 288, 2, 5, 20000),
    (200, 288, 1, 5, 20000),
    (500, 992, 1, 1, 30000),
    (500, 992, 2, 4, 30000),
    (1000, 1440, 2, 5, 30000),
    (1000, 1440, 1, 1, 30000),
    (2000, 2944, 2, 2, 40000),
    (2000, 4096, 1, 1, 40000),
]


@pytest.mark.parametrize("ascending", [False, True])
@pytest.mark.parametrize("k,kp,cg,ns,n", CONTRACT_CASES)
def test_candidate_contract(k, kp, cg, ns, n, ascending):
    d = 256
    Q = _ln_rows(np.random.default_rng(11), 130, d)      # 130: a ragged query tile for CG 1 and 2
    P = _ties_corpus(n, d, Q[0], kp, seed=kp + n, ascending=ascending)
    idx = _make(P, "fp16", kprime=kp, cta_group=cg, n_splits=ns, tier2=0, exact_fallback=0)
    D, I = idx.search(Q, k)
    C = _coarse_scores(idx, Q.shape[0], n, d, "fp16", cg)
    ps = _check_contract(idx, C, n)
    assert ps["tier"] == 1 and ps["kprime"] == kp and ps["nq"] == 130
    if not ascending and ns == 1:
        eq = (C[0, 40:40 + 3 * 48:3] == C[0, 40]).all()
        thr0 = torch.from_numpy(_state(idx, "cand_thr", (130, 1), torch.float32))[0, 0]
        assert eq and C[0, 40].item() == thr0.item(), "the planted ties do not straddle the cut"
    # queries tier 1 certified are exact
    nf = int(_state(idx, "flagged_cnt", 1, torch.int32)[0])
    flagged = set(_state(idx, "flagged", nf, torch.int32).tolist())
    ok = np.array([q not in flagged for q in range(130)])
    Do, Io = flat_ip_oracle.search(P, Q, k)
    assert (I[ok] == Io[ok]).all() and (D[ok] == Do[ok]).all()


def test_tier2_keeps_every_row_above_its_start_threshold():
    """bf16 with k' = k + 32: tier 1 fails for most queries; tier 2 (exact_fallback = 0) keeps, per flagged query and
    split, every row whose coarse score exceeds its start threshold unless the reservoir compacted."""
    d, n, k = 256, 60000, 200
    P = _ln_rows(np.random.default_rng(21), n, d)
    Q = _ln_rows(np.random.default_rng(22), 130, d)
    idx = _make(P, "bf16", kprime=k + 24, n_splits=1, exact_fallback=0)
    idx.search(Q, k)
    nf = int(_state(idx, "flagged_cnt", 1, torch.int32)[0])
    assert nf >= 20
    flagged = _state(idx, "flagged", nf, torch.int32)
    fthr = torch.from_numpy(_state(idx, "flagged_thr", nf, torch.float32)).cuda()
    ps = _pass(idx)
    assert ps["tier"] == 2 and ps["nq"] == nf
    qsel = torch.from_numpy(flagged.astype(np.int64)).cuda()
    # the tier-2 pass's coarse scores: the rows of Q16 it gathered, against P16
    q16 = torch.from_numpy(_state(idx, "q16", (130, d), torch.int16)).cuda()[qsel]
    p16 = torch.from_numpy(_state(idx, "p16", (n, d), torch.int16)).cuda()
    C = torch.empty((nf, n), device="cuda")
    _lib.check(_lib.load().ance_dbg_gemm(q16.contiguous().data_ptr(), p16.data_ptr(), nf, n, d, 1, 2, None, None, 0,
                                         None, C.data_ptr(), _lib.current_stream()))
    torch.cuda.synchronize()
    _check_contract(idx, C, n, thr_floor=fthr)


# ---------------------------------------------------------------------------------------------------------------------
# 3. corpora that defeat a bound that is too small
# ---------------------------------------------------------------------------------------------------------------------
FAMILIES = {
    # name: corpus kwargs, k, k'
    "row_fp16_768": (dict(fmt="fp16", d=768), 100, 160),
    "row_bf16_256": (dict(fmt="bf16", d=256), 100, 256),
    "query_bf16_768": (dict(fmt="bf16", d=768, mode="query"), 100, 256),
    "centred_fp16_768": (dict(fmt="fp16", d=768, center=True), 100, 160),
    "large_k_fp16_768": (dict(fmt="fp16", d=768, nq=12, n_background=4000), 1000, 1440),
}


@functools.lru_cache(maxsize=None)
def _family(name):
    args, k, kp = FAMILIES[name]
    args = {"nq": 32, "n_background": 3000, **args}
    c = sr.residual_corpus(k=k, kprime=kp, seed=5, **args)
    Do, Io = flat_ip_oracle.search_bruteforce(c["P"], c["Q"], k)
    return c, k, kp, Do, Io


CASES = [(f, False) for f in FAMILIES] + [("row_fp16_768", True), ("centred_fp16_768", True), ("query_bf16_768", True)]


@pytest.mark.parametrize("name,host", CASES)
def test_tier1_flags_every_wrong_answer(name, host):
    c, k, kp, Do, Io = _family(name)
    P, Q, fmt = c["P"], c["Q"], c["fmt"]
    nq, d = Q.shape
    idx = _make(P, fmt, host, kprime=kp, n_splits=1, tier2=0, exact_fallback=0, center=int(c["mu"] is not None))
    D, I = idx.search(Q, k)
    wrong = (I != Io).any(1) | (D != Do).any(1)
    nf = int(_state(idx, "flagged_cnt", 1, torch.int32)[0])
    flagged = np.zeros(nq, bool)
    flist = _state(idx, "flagged", nf, torch.int32)
    flagged[flist] = True
    assert wrong.sum() >= nq // 2, f"only {wrong.sum()} of {nq} tier-1 answers are wrong: the corpus lost its strength"
    assert flagged[wrong].all(), f"queries {np.flatnonzero(wrong & ~flagged)} are wrong and certified"
    assert (I[~flagged] == Io[~flagged]).all() and (D[~flagged] == Do[~flagged]).all()
    # the decision, recomputed in fp64 from the exported threshold, the kernel's scores and norms
    centred = bool(_state(idx, "centred", 1, torch.int32)[0])
    mu = _state(idx, "mu", d, torch.float32) if centred else None
    if c["mu"] is not None:
        assert centred and (mu == c["mu"]).all()          # mirrored rows: the index centres on exactly m
    thr = _state(idx, "cand_thr", (nq, 1), torch.float32)[:, 0]
    ps = _state(idx, "pstats", 2, torch.float32).astype(np.float64)
    qn = _state(idx, "qn_hat", nq, torch.float32)
    qd = _state(idx, "qn_delta", nq, torch.float32)
    qmu = np.zeros(nq) if mu is None else Q.astype(np.float64) @ mu.astype(np.float64)
    eps_k = sr.eps_bound(qn, qd, ps[0], ps[1], d)
    cert, _ = sr.certificate(thr, D[:, k - 1], eps_k, qmu)
    margin = np.abs(thr + eps_k + qmu - D[:, k - 1] * (1 - 1.2e-7))
    sure = margin > 1e-5 * eps_k
    assert (cert[sure] == ~flagged[sure]).all()
    # tier 2 would start low enough: at or below the fp64 threshold of exact norms
    _, hat, _ = sr.operand_rows(P, mu, fmt)
    _, qhat = sr.round16(Q, fmt)
    pn, pd, _ = sr.exact_norms(P, mu, hat)
    qn_x, qd_x, _ = sr.exact_norms(Q, None, qhat)
    _, nxt = sr.certificate(thr, D[:, k - 1], sr.eps_bound(qn_x, qd_x, pn.max(), pd.max(), d, factor=1.0), qmu)
    fthr = _state(idx, "flagged_thr", nf, torch.float32)
    assert (fthr <= nxt[flist]).all()
    ratio = (D[:, k - 1].astype(np.float64) * (1 - 1.2e-7) - thr - qmu) / eps_k
    worst = ratio[wrong].max()
    print(f"{name} host={host}: {wrong.sum()}/{nq} wrong at tier 1, all flagged; eps {eps_k.max():.4f}, "
          f"max (s_k_lo - thr - <q,mu>) / eps over wrong queries {worst:.3f}")
    assert worst >= 0.5
    if host:
        st = idx.stats()
        assert 0 < idx.last_fetched() < st["n_candidates"], (idx.last_fetched(), st)


@pytest.mark.parametrize("n_splits", [0, 1])
@pytest.mark.parametrize("name,host", CASES)
def test_default_search_is_exact_on_adversarial_corpora(name, host, n_splits):
    """Default parameters but the family's centring (the uncentred families are built for center = 0; centred on the
    column mean their residuals are no longer aligned): n_splits = 0 (automatic; with row-range splits the hidden rows
    are candidates of their own split), and one sweep per query (n_splits = 1), where tier 1 fails for every query and
    tier 2 must recover."""
    c, k, kp, Do, Io = _family(name)
    idx = _make(c["P"], c["fmt"], host, n_splits=n_splits, center=int(c["mu"] is not None))
    D, I = idx.search(c["Q"], k)
    assert (I == Io).all() and (D.view(np.uint32) == Do.view(np.uint32)).all()
    st = idx.stats()
    print(f"{name} host={host} n_splits={st['n_splits']}: tier 2 {st['n_tier2']}, brute force {st['n_uncertified']} "
          f"of {st['nq']}")
    if n_splits == 1:
        assert st["n_tier2"] == st["nq"], st


def test_zero_scores_tie_across_splits():
    """Rows whose support is disjoint from the queries' score exactly 0 (+0 and -0 components) and sit at the rank-k
    boundary in every split: the answer is the oracle's, ties in ascending row order."""
    d, n, k = 256, 12000, 100
    rng = np.random.default_rng(31)
    Q = np.zeros((64, d), np.float32)
    Q[:, : d // 2] = rng.standard_normal((64, d // 2))
    P = np.zeros((n, d), np.float32)
    P[:, d // 2:] = rng.standard_normal((n, d // 2))                      # score 0 against every query
    P[::7, d // 2:] *= -1.0
    P[::97, : d // 2] = np.abs(rng.standard_normal((len(range(0, n, 97)), d // 2))) * np.sign(Q[0, : d // 2])
    P[1::13, : d // 2] = -0.0
    Do, Io = flat_ip_oracle.search_bruteforce(P, Q, k)
    for host in (False, True):
        idx = _make(P, "fp16", host, n_splits=8)
        D, I = idx.search(Q, k)
        assert (I == Io).all() and (D.view(np.uint32) == Do.view(np.uint32)).all()
        idx1 = _make(P, "fp16", host, n_splits=8, tier2=0, exact_fallback=0)
        idx1.search(Q, k)
        C = _coarse_scores(idx1, 64, n, d, "fp16", 2)
        _check_contract(idx1, C, n)
