"""CPU checks of tests/search_refs.py: the references restate the kernels' arithmetic, the norm bounds cover an fp32
emulation of quantize_rows_kernel, and the adversarial corpora discriminate: with the full eps the tier-1 emulation
certifies no wrong answer, with a residual term dropped or halved it certifies wrong ones."""
import numpy as np
import pytest
import torch

from tests import search_refs as sr

FAMILIES = {
    # name: (corpus kwargs, k, k', the eps term the corpus is built against)
    "row_fp16_768": (dict(fmt="fp16", d=768), 100, 160, "qn_maxdp"),
    "row_bf16_256": (dict(fmt="bf16", d=256), 100, 256, "qn_maxdp"),
    "query_bf16_768": (dict(fmt="bf16", d=768, mode="query"), 100, 256, "qd_maxp"),
    "centred_fp16_768": (dict(fmt="fp16", d=768, center=True), 100, 160, "qn_maxdp"),
}


def _corpus(name, **kw):
    args, k, kp, term = FAMILIES[name]
    c = sr.residual_corpus(nq=16, k=k, kprime=kp, n_background=1000, seed=3, **{**args, **kw})
    return c, k, kp, term


def test_round16_is_rne_at_the_edges():
    x = np.array([65504.0, -65504.0, 65519.0, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11,
                  1e-30, -0.0], dtype=np.float32)
    bits, v = sr.round16(x, "fp16")
    assert (v == torch.from_numpy(x).half().double().numpy()).all()
    assert (sr.bits_to_f64(bits, "fp16") == v).all()
    assert v[2] == 65504.0 and v[4] == 0.0 and v[5] == 2.0 ** -24 and v[6] == 1.0 and v[7] == 1.0 + 2.0 ** -9
    bits, v = sr.round16(x, "bf16")
    assert (sr.bits_to_f64(bits, "bf16") == v).all()
    assert v[6] == 1.0 and np.signbit(v[-1])


def test_mirrored_rows_have_an_exact_mean():
    c, *_ = _corpus("centred_fp16_768")
    assert (sr.mean_ref(c["P"]) == c["mu"]).all()
    _, hat, X = sr.operand_rows(c["P"], c["mu"], "fp16")
    n = c["P"].shape[0] // 2
    assert (X[:n] == -X[n:]).all()                        # fl32(p - mu) = +-v exactly


def _quantize_emulation(X: np.ndarray, fmt: str):
    """quantize_rows_kernel in fp32: lane l sums elements l*4 + 128 t .. + 3 with fmaf, then the xor-shuffle tree."""
    n, d = X.shape
    _, hat = sr.round16(X, fmt)
    hat32 = hat.astype(np.float32)
    e = (X - hat32).astype(np.float32)
    sums = []
    for v in (hat32, e, X):
        lanes = np.zeros((n, 32), np.float32)
        for t0 in range(0, d, 128):
            for u in range(4):
                cols = t0 + np.arange(32) * 4 + u
                ok = cols < d
                a = v[:, np.minimum(cols, d - 1)].astype(np.float64)
                lanes = np.where(ok[None, :], (a * a + lanes).astype(np.float32), lanes)
        for s in (16, 8, 4, 2, 1):
            lanes = (lanes + lanes[:, np.arange(32) ^ s]).astype(np.float32)
        sums.append(lanes[:, 0])
    sh, sd, sx = sums
    nh = (np.sqrt(sh) * np.float32(1.00001)).astype(np.float32)
    return nh, sd, sx


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
@pytest.mark.parametrize("centred", [False, True])
def test_norm_bounds_cover_the_kernel_arithmetic(fmt, centred):
    rng = np.random.default_rng(4)
    d = 256
    P = rng.standard_normal((400, d)).astype(np.float32) * np.float32(3.0)
    P[0] = 60000.0 if fmt == "fp16" else 1e17             # near the top of the range (bf16: of its squared norm)
    P[1] = 1e-6                                           # fp16 subnormal range: the relative residual is large
    P[2, :] = 0.7                                         # constant row
    P[3] = rng.standard_normal(d) * 1e-4
    mu = sr.mean_ref(P) if centred else None
    _, hat, X = sr.operand_rows(P, mu, fmt)
    nh, sd, sx = _quantize_emulation(X, fmt)
    nd = ((np.sqrt(sd) + (np.float32(1.2e-7) * np.sqrt(sx) if centred else np.float32(0)))
          * np.float32(1.00001)).astype(np.float32)
    pn, pd, xn = sr.exact_norms(P, mu, hat)
    assert (nh >= pn).all() and (nh <= sr.norm_upper(pn, xn, d, False)).all()
    assert (nd >= pd).all() and (nd <= sr.norm_upper(pd, xn, d, centred)).all()


def test_certificate_reference_rules():
    cert, nxt = sr.certificate([-np.inf, 1.0, 1.0], [5.0, 5.0, 5.0], [0.5, 3.9, 4.1], [0.0, 0.0, 0.0])
    assert cert.tolist() == [True, True, False]
    assert nxt[2] < 5.0 - 4.1
    e = sr.eps_bound(2.0, 0.5, 3.0, 0.25, 768, factor=1.0)
    assert e == pytest.approx(0.5 * 3 + 2 * 0.25 + 0.5 * 0.25 + 768 * 2.0 ** -22 * 2 * 3, rel=1e-15)
    assert sr.eps_bound(2.0, 0.5, 3.0, 0.25, 768, {"qd_maxp": 0}, factor=1.0) == pytest.approx(e - 1.5, rel=1e-15)


@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_corpus_defeats_a_bound_that_is_too_small(name):
    c, k, kp, term = _corpus(name)
    full = sr.emulate(c, k, kp)
    # every query's tier-1 answer is wrong, and the full bound refuses to certify any of them
    assert full["wrong"].all()
    assert not (full["certified"] & full["wrong"]).any()
    assert full["ratio"][full["wrong"]].max() >= 0.5
    for f in (0.0, 0.5):
        bad = sr.emulate(c, k, kp, scale={term: f})
        assert (bad["certified"] & bad["wrong"]).sum() >= 1, (name, term, f)
    # the structure the GPU tests rely on: the hidden rows are just below the tier-1 threshold, the fillers are candidates
    Ch = full["Chat"]
    for i in range(c["Q"].shape[0]):
        assert (Ch[i, c["hidden"][i]] < full["thr"][i]).all()
        assert np.isin(c["fillers"][i], full["cands"][i]).all()


def test_prefilter_drops_a_hidden_row_with_the_next_rows_residual_norm():
    """The host pre-filter with the exact per-row residual norms keeps every row of the true top k; reading row j + 1's
    norm for row j (the hidden rows' neighbours carry no residual) drops hidden rows that belong to it."""
    c, k, kp, _ = _corpus("row_fp16_768")
    e = sr.emulate(c, k, kp)
    P, Q = c["P"], c["Q"]
    nd = e["pd"] * (1 + 1e-6)
    nd_next = np.concatenate([nd[1:], nd[:1]])
    maxp, maxdp = e["pn"].max(), e["pd"].max()
    truth = sr.true_topk(e["S"], k)
    _, nxt = sr.certificate(e["thr"], e["D"][:, k - 1], e["eps"], e["qmu"])
    lost = 0
    for i in range(Q.shape[0]):
        rows = np.flatnonzero(e["Chat"][i] > nxt[i])       # tier 2's candidates: every row above its threshold
        assert np.isin(truth[i], rows).all()
        keep = sr.prefilter(Q[i], rows, e["phat"], nd, None, maxp, maxdp, k)
        assert np.isin(truth[i], rows[keep]).all() and keep.sum() < len(rows)
        keep2 = sr.prefilter(Q[i], rows, e["phat"], nd_next, None, maxp, maxdp, k)
        lost += int(not np.isin(truth[i], rows[keep2]).all())
    assert lost >= 1
