"""fp64 references of the flat-IP search's exactness certificate, and corpora on which a bound that is too small gives a
wrong answer (test infrastructure only).

The search is exact by proof, not by tolerance (search.cu, rescore_kernel): a row that is not a candidate has centred
coarse score <= thr, hence exact score <= thr + eps(q) + <q, mu>; when that is below the k-th exact score found, the
answer is the exact top k.  Everything below restates the proof's inputs and its two inequalities in fp64, from the
kernel's own exported state (ance_dbg_index_state), with these bounds:

* mu: ``fl32(sum_fp64(x) / n)``.  The kernel adds per-block fp64 partial sums with atomics in no fixed order, so its mu is
  within 1 ulp32 of the reference (the fp64 sums differ by far less than half an fp32 ulp; only the final rounding can
  land on the other side of a midpoint).
* Operand rows: ``p^ = RNE16(fl32(p - mu_kernel))``, bit for bit (fp16 through numpy, bf16 through torch's CPU RNE).
* Norms: with x = fl32(p - mu), e = x - p^ and the exact residual delta = (p - mu) - p^ (p - mu exact in fp64), the
  kernel stores ``nd = (||e||_32 + 1.2e-7 ||x||_32) * 1.00001`` (``_32``: lane-strided fp32 sums of squares, relative
  error below (d/32 + 8) 2^-24, then sqrt).  Since ||delta|| <= ||e|| + ||x - (p - mu)|| <= ||e|| + 2^-24 ||x||:
  ``||delta|| <= nd <= (||delta|| + (2^-24 + 1.2e-7) ||x||) (1 + (d/32 + 8) 2^-24) 1.00001 (1 + 2^-22)``.
  ||p^|| and the query norms likewise, without the subtraction term (queries are not centred).
* The certificate: ``eps = (qd maxp + qn maxdp + qd maxdp + d 2^-22 qn maxp) 1.0001`` from the kernel's norms, and
  certified iff ``thr + eps + <q, mu>(1 + 1e-12) < s_k (1 - 1.2e-7)`` (s_k the kernel's k-th score).  The next tier
  starts below ``s_k_lo - <q, mu> - eps_exact``, eps_exact the same expression of exact norms without the 1.0001.
* The host pre-filter: ``lo_j / hi_j = <q, mu> + s~_j -/+ (||q|| nd_j (1 + (d + 64) 2^-23) + g)`` with
  ``g = (d + 16) 2^-53 ||q|| (||mu|| + maxp + maxdp)``; row j is dropped iff ``hi_j + g < L - g``, L the k-th largest lo.
  Evaluated in fp64 without the kernel's directed roundings (they move the bounds by ~1e-16 relative).

The tier-1 emulation rebuilds the coarse pass from exact dots of the 16-bit operands (the corpora below keep every coarse
score on a grid that fp32 holds exactly, so the tensor core's summation order cannot matter) and a stable top-k' per
split, then applies the certificate with eps made of separately scalable terms.  Dropping or halving a term shows which
corpora discriminate.  Two parts of the bound are too small to show on any corpus the certificate can see: the g term of
the pre-filter (~1e-13 of ||q|| ||p||) and the directed roundings, and the ``1.2e-7 ||x||`` subtraction term next to the
accumulation term (d 2^-22 = 1.8e-4 at d = 768, 1,500x larger).

Corpora (``residual_corpus``): queries are sign vectors, rows have entries of magnitude in [1.0625, 2), so every product
and partial sum lies on a grid of 2^-10 (fp16) / 2^-7 (bf16) and the coarse scores are exact in fp32.  Per query: k - 1
clear winners, k' - k + 1 residual-free fillers with coarse scores in [x, x + c], and hidden rows at coarse x - ulp whose
fp32 rows carry a residual aligned with the query (mode "row": +h sign(q) per element, h just under half an ulp, so the
exact score exceeds the coarse one by R = d h), or, with exact rows, a query residual aligned with the hidden row and
opposite to the fillers (mode "query").  Tier 1 keeps the fillers, its answer is wrong, and only the part of eps that
covers the residual keeps the certificate from accepting it.  This needs one sweep per query (n_splits = 1): with
row-range splits every split keeps its own k' best rows, the hidden rows become candidates and tier 1 is right.
``center=True`` mirrors every row about a common vector m ((m + v, m - v) on grids where fp64 column sums and
fl32(p - m) are exact): mu = m and the centred rows are exactly v.
"""
from __future__ import annotations

import numpy as np
import torch

F64 = np.float64
U32 = 2.0 ** -24
ULP = {"fp16": 2.0 ** -10, "bf16": 2.0 ** -7}   # spacing of the 16-bit format on [1, 2)
EPS_TERMS = ("qd_maxp", "qn_maxdp", "qd_maxdp", "accum")


# ---------------------------------------------------------------------------------------------------------------------
# operands and norms
# ---------------------------------------------------------------------------------------------------------------------
def round16(x: np.ndarray, fmt: str):
    """RNE of fp32 values to the 16-bit format: (bits uint16, values fp64)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    if fmt == "fp16":
        h = x.astype(np.float16)
        return h.view(np.uint16), h.astype(F64)
    t = torch.from_numpy(x).to(torch.bfloat16)
    return t.view(torch.int16).numpy().view(np.uint16), t.to(torch.float64).numpy()


def bits_to_f64(bits: np.ndarray, fmt: str) -> np.ndarray:
    bits = np.ascontiguousarray(bits).view(np.uint16)
    if fmt == "fp16":
        return bits.view(np.float16).astype(F64)
    return (bits.astype(np.uint32) << 16).view(np.float32).astype(F64)


def mean_ref(P: np.ndarray) -> np.ndarray:
    """fl32(sum_fp64(x) / n) per column."""
    return (P.astype(F64).sum(0) / P.shape[0]).astype(np.float32)


def ulp32(x: np.ndarray) -> np.ndarray:
    x = np.abs(np.asarray(x, dtype=np.float32))
    return np.spacing(np.maximum(x, np.float32(2.0 ** -126))).astype(F64)


def operand_rows(P: np.ndarray, mu, fmt: str):
    """Kernel-exact operands of index rows (mu: the kernel's centre, or None): (bits, p^ fp64, x = fl32(p - mu))."""
    X = P if mu is None else (P - mu[None, :]).astype(np.float32)
    bits, hat = round16(X, fmt)
    return bits, hat, X


def exact_norms(P: np.ndarray, mu, hat: np.ndarray):
    """(||p^||, ||(p - mu) - p^||, ||x||) in fp64, p - mu exact."""
    C = P.astype(F64) - (0.0 if mu is None else mu.astype(F64)[None, :])
    return np.sqrt((hat * hat).sum(1)), np.sqrt(((C - hat) ** 2).sum(1)), np.sqrt((C * C).sum(1))


def norm_upper(exact: np.ndarray, xnorm: np.ndarray, d: int, centred: bool) -> np.ndarray:
    """Largest value the kernel may store for a norm whose exact value is `exact` (module docstring)."""
    sub = (U32 + 1.2e-7) * xnorm if centred else 0.0
    return (exact + sub) * (1.0 + (d / 32 + 8) * U32) * 1.00001 * (1.0 + 2.0 ** -22) + 1e-30


# ---------------------------------------------------------------------------------------------------------------------
# the certificate and the pre-filter
# ---------------------------------------------------------------------------------------------------------------------
def eps_bound(qn, qd, maxp, maxdp, d: int, scale=None, factor: float = 1.0001):
    """eps(q) of rescore_kernel in fp64; scale: {term: factor} to drop (0) or shrink a term (see EPS_TERMS)."""
    s = {t: 1.0 for t in EPS_TERMS}
    s.update(scale or {})
    qn, qd = np.asarray(qn, F64), np.asarray(qd, F64)
    e = (s["qd_maxp"] * qd * maxp + s["qn_maxdp"] * qn * maxdp + s["qd_maxdp"] * qd * maxdp
         + s["accum"] * d * 2.0 ** -22 * qn * maxp)
    return e * factor


def certificate(thr, sk, eps, qmu):
    """(certified, next-tier threshold) of rescore_kernel, in fp64.  thr: max over splits of cand_thr; sk: the k-th
    score (fp32); eps from eps_bound; qmu = <q, mu> (0 when not centred)."""
    thr, sk, eps, qmu = (np.asarray(a, F64) for a in (thr, sk, eps, qmu))
    qmu_up = qmu + np.abs(qmu) * 1e-12
    sk_lo = sk - np.abs(sk) * 1.2e-7
    cert = np.where(np.isneginf(thr), True, thr + eps + qmu_up < sk_lo)
    return cert, sk_lo - qmu - eps


def prefilter(q: np.ndarray, rows: np.ndarray, hat: np.ndarray, nd: np.ndarray, mu, maxp: float, maxdp: float, k: int):
    """Survivor mask of host_rows_scores over candidate rows `rows` of query q (fp32): hat = p^ of all rows (fp64), nd =
    the per-row residual norms the pre-filter reads."""
    d = q.shape[0]
    q64 = q.astype(F64)
    qn = np.sqrt((q64 * q64).sum() * (1.0 + (d + 16) * 2.0 ** -52))
    mun = 0.0 if mu is None else float(np.sqrt((mu.astype(F64) ** 2).sum()))
    qmu = 0.0 if mu is None else float(q64 @ mu.astype(F64))
    g = (d + 16) * 2.0 ** -53 * qn * (mun + maxp + maxdp)
    st = hat[rows] @ q64
    r = qn * nd[rows] * (1.0 + (d + 64) * 2.0 ** -23) + g
    lo, hi = qmu + st - r, qmu + st + r
    if len(rows) <= k:
        return np.ones(len(rows), bool)
    L = np.sort(lo)[::-1][k - 1]
    return hi + g >= L - g


# ---------------------------------------------------------------------------------------------------------------------
# tier-1 emulation
# ---------------------------------------------------------------------------------------------------------------------
def topk_rows(scores: np.ndarray, rows: np.ndarray, k: int) -> np.ndarray:
    """The k best of `rows` by (score desc, row asc)."""
    o = np.lexsort((rows, -scores))
    return rows[o[:k]]


def exact_scores(Q: np.ndarray, P: np.ndarray) -> np.ndarray:
    """fp32-input dot products accumulated in fp64, rounded once to fp32 (the oracle's and the kernel's scores)."""
    return (Q.astype(F64) @ P.astype(F64).T).astype(np.float32)


def tier1(Chat: np.ndarray, S: np.ndarray, k: int, kprime: int, rows_per_split: int):
    """Tier 1 on exact coarse scores Chat [nq, n] (fp64 of the 16-bit operands) and exact scores S [nq, n] (fp32):
    per split the stable top k' (thr = its k'-th coarse score, -inf when the split has <= k' rows), then the top k of the
    candidates by exact score.  Returns (thr [nq], I [nq, k], D [nq, k], candidates list)."""
    nq, n = Chat.shape
    thr = np.full(nq, -np.inf)
    I = np.zeros((nq, k), np.int64)
    cands = []
    for i in range(nq):
        cs = []
        for r0 in range(0, n, rows_per_split):
            rows = np.arange(r0, min(n, r0 + rows_per_split))
            top = topk_rows(Chat[i, rows], rows, kprime)
            if len(rows) > kprime:
                thr[i] = max(thr[i], Chat[i, top[-1]])
            cs.append(top)
        c = np.concatenate(cs)
        cands.append(c)
        I[i] = topk_rows(S[i, c].astype(F64), c, k)
    return thr, I, np.take_along_axis(S, I, 1), cands


def true_topk(S: np.ndarray, k: int) -> np.ndarray:
    rows = np.arange(S.shape[1])
    return np.stack([topk_rows(S[i].astype(F64), rows, k) for i in range(S.shape[0])])


def emulate(corpus: dict, k: int, kprime: int, rows_per_split=None, scale=None):
    """The whole tier-1 decision on a corpus, on the CPU.  Returns per query: wrong (tier 1's top k differs from the
    exact one), certified, the ratio (s_k_lo - thr - <q, mu>) / eps, and the pieces."""
    fmt, P, Q, mu = corpus["fmt"], corpus["P"], corpus["Q"], corpus["mu"]
    d = P.shape[1]
    _, phat, _ = operand_rows(P, mu, fmt)
    _, qhat = round16(Q, fmt)
    pn, pd, _ = exact_norms(P, mu, phat)
    qn, qd, _ = exact_norms(Q, None, qhat)
    Chat = qhat @ phat.T
    S = exact_scores(Q, P)
    thr, I, D, cands = tier1(Chat, S, k, kprime, rows_per_split or P.shape[0])
    eps = eps_bound(qn, qd, pn.max(), pd.max(), d, scale)
    qmu = np.zeros(Q.shape[0]) if mu is None else Q.astype(F64) @ mu.astype(F64)
    cert, _ = certificate(thr, D[:, k - 1], eps, qmu)
    wrong = (I != true_topk(S, k)).any(1)
    ratio = (D[:, k - 1].astype(F64) * (1 - 1.2e-7) - thr - qmu) / eps
    return dict(wrong=wrong, certified=cert, ratio=ratio, thr=thr, I=I, D=D, eps=eps, cands=cands, Chat=Chat, S=S,
                phat=phat, pd=pd, pn=pn, qn=qn, qd=qd, qmu=qmu)


# ---------------------------------------------------------------------------------------------------------------------
# corpora
# ---------------------------------------------------------------------------------------------------------------------
A = 1.0625   # smallest row magnitude: |p^_j| in [A, 2), one ulp both ways


def _row(rng, s: np.ndarray, target: float, ulp: float, free=None) -> np.ndarray:
    """A 16-bit-exact row v with <s, v> == target exactly: entries s_j f_j (A + m_j ulp), f = +-1.  free: the coordinates
    that may vary (others are left 0 for the caller to fill)."""
    d = s.shape[0]
    free = np.arange(d) if free is None else free
    nf = len(free)
    nflip = int(np.ceil((nf - target / A) / 2))          # A (nf - 2 nflip) <= target
    assert 0 <= nflip < nf // 2, (target, nf)
    f = np.ones(nf)
    f[rng.choice(nf, nflip, replace=False)] = -1.0
    M = int(round((target - A * f.sum()) / ulp))
    assert M >= 0 and abs(A * f.sum() + M * ulp - target) == 0.0
    m = np.zeros(nf)
    pos = np.flatnonzero(f > 0)
    cap = int(0.7 / ulp)
    share = rng.permutation(pos)
    for j in share:                                       # spread the remainder, at most 0.7 per entry
        t = min(M, cap)
        m[j] += t
        M -= t
        if M == 0:
            break
    assert M == 0
    v = np.zeros(d)
    v[free] = s[free] * f * (A + m * ulp)
    return v


def residual_corpus(fmt: str = "fp16", d: int = 768, nq: int = 32, k: int = 100, kprime: int = 160, n_hidden: int = 2,
                    n_background: int = 2000, mode: str = "row", center: bool = False, seed: int = 0) -> dict:
    """Rows and queries of the module docstring.  Returns dict(P, Q fp32, mu (the centre the index must find, or None),
    fmt, hidden [nq, n_hidden] row numbers, fillers [nq, k' - k + 1], R (the score each hidden row hides))."""
    rng = np.random.default_rng(seed)
    ulp = ULP[fmt]
    S = rng.choice([-1.0, 1.0], size=(nq, d))
    x = np.round(0.5 * A * d / ulp) * ulp if mode == "row" else np.round(0.25 * A * d / ulp) * ulp
    nfill = kprime - k + 1
    rows, hidden, fillers = [], [], []
    if mode == "row":
        h = ulp / 2 - 2.0 ** -20                # just under half an ulp: the residual rounds away
        R = d * h
        gap = R                                 # hidden exact - hidden coarse
        c = np.floor((R - 3 * ulp) / ulp) * ulp
    else:
        g = ulp / 4 - 2.0 ** -20                # under half the spacing just below 1 (ulp / 2): q^ = sign(q)
        half = d // 2
        R = None
    Q = S.copy()
    for i in range(nq):
        s = S[i]
        if mode == "query":
            Sset = np.sort(rng.choice(d, half, replace=False))
            T = np.setdiff1d(np.arange(d), Sset)
            fH = np.ones(half)
            fH[rng.choice(half, half // 2, replace=False)] = -1.0      # sum over the set: 0
            hs = s[Sset] * fH * A                                      # the hidden rows' entries on the set
            G = g * A * half
            R = 2 * G                                                  # hidden gains G, fillers lose G
            gap = G
            c = np.floor((2 * G - 3 * ulp) / ulp) * ulp
            Q[i, Sset] = s[Sset] + g * np.sign(hs)
        top = np.round((x + (R if mode == "row" else G) + 4.0) / ulp) * ulp
        for j in range(k - 1):                                         # winners
            rows.append(_row(rng, s, top + np.round(0.05 * j / ulp) * ulp, ulp))
        fl = []
        for t in range(nfill):                                         # residual-free fillers on [x, x + c]
            tgt = x + np.round(c * t / max(1, nfill - 1) / ulp) * ulp
            if mode == "row":
                v = _row(rng, s, tgt, ulp)
            else:
                v = _row(rng, s, tgt, ulp, free=T)
                v[Sset] = -hs
            fl.append(len(rows))
            rows.append(v)
        hd = []
        for _ in range(n_hidden):                                      # hidden rows at coarse x - ulp
            if mode == "row":
                v = _row(rng, s, x - ulp, ulp) + h * s
            else:
                v = _row(rng, s, x - ulp, ulp, free=T)
                v[Sset] = hs
            hd.append(len(rows))
            rows.append(v)
        fillers.append(fl)
        hidden.append(hd)
    for _ in range(n_background):                                      # exact, no longer than the structured rows
        rows.append(A * rng.choice([-1.0, 1.0], size=d))
    V = np.stack(rows)
    perm = rng.permutation(len(rows))                                  # spread every structure over the corpus
    inv = np.argsort(perm)
    V = V[perm]
    hidden = inv[np.array(hidden)]
    fillers = inv[np.array(fillers)]
    mu = None
    if center:
        m = np.round(rng.uniform(-8, 8, size=d) * 16) / 16             # |m| <= 8 on a 2^-4 grid: m +- v exact in fp32
        V = np.concatenate([m + V, m - V])
        mu = m.astype(np.float32)
    P = V.astype(np.float32)
    assert (P.astype(F64) == V).all(), "rows not exact in fp32"
    Qf = Q.astype(np.float32)
    assert (Qf.astype(F64) == Q).all()
    return dict(P=P, Q=Qf, mu=mu, fmt=fmt, hidden=hidden, fillers=fillers, R=R, gap=gap, x=x, c=c, k=k, kprime=kprime)
