"""Searches with 512 < k <= 2048 (top-1000 full-rank evaluation, large --topk_training): the large-k path (8192-entry
reservoirs, streaming compaction, query blocks) and the brute force at those sizes, bit-exact (int64 labels and fp32
scores) against the CPU oracle."""
import functools

import numpy as np
import pytest
import torch

from oracle import flat_ip_oracle
from tests.test_gpu_search import _index, _ln_rows

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _world():
    P = _ln_rows(np.random.default_rng(1234), 60000, 768)
    Q = _ln_rows(np.random.default_rng(4321), 300, 768)
    return P, Q


@functools.lru_cache(maxsize=None)
def _oracle(k):
    P, Q = _world()
    return flat_ip_oracle.search(P, Q, k)


def _same(D, I, Do, Io):
    assert (I == Io).all(), f"{(I != Io).any(1).sum()} queries differ"
    assert (D.view(np.uint32) == Do.view(np.uint32)).all()


@pytest.mark.parametrize("operand", ["bf16", "fp16"])
@pytest.mark.parametrize("cta_group", [1, 2])
@pytest.mark.parametrize("k", [513, 1000, 1024, 2048])
def test_seeded_parity_large_k(operand, cta_group, k):
    P, Q = _world()
    idx = _index(P, operand, cta_group=cta_group)
    D, I = idx.search(Q, k)
    _same(D, I, *_oracle(k))
    st = idx.stats()
    assert st["nq"] == 300 and st["kprime"] > 992 and st["kprime"] >= k, st
    if operand == "fp16" and k in (1000, 2048):
        assert st["n_uncertified"] == 0, st      # certified by the coarse path, not produced by the brute force


def test_query_counts_and_whole_corpus_sweeps_at_1000():
    P, Q = _world()
    k = 1000
    Do, Io = _oracle(k)
    idx = _index(P)
    for nq in (1, 7, 300):
        D, I = idx.search(Q[:nq], k)
        _same(D, I, Do[:nq], Io[:nq])
        assert idx.stats()["nq"] == nq
    assert idx.stats()["n_splits"] > 1           # 300 queries are two query tiles: the corpus is split into row ranges
    # four clusters of two CTAs and 2048 queries (eight query tiles): every work item sweeps the whole corpus
    Q2 = _ln_rows(np.random.default_rng(77), 2048, 768)
    idx2 = _index(P, "fp16", max_ctas=8)
    D, I = idx2.search(Q2, k)
    assert idx2.stats()["n_splits"] == 1
    _same(D, I, *flat_ip_oracle.search(P, Q2, k))


def test_tier2_forced_large_k():
    """bf16 operands (eps ~ 3) with k' barely above k: tier 1 cannot certify, tier 2 restarts from the thresholds."""
    P, Q = _world()
    k = 1000
    idx = _index(P, "bf16", kprime=1024, n_splits=1)
    D, I = idx.search(Q, k)
    st = idx.stats()
    assert st["n_tier2"] > 0 and st["kprime"] == 1024, st
    _same(D, I, *_oracle(k))


@pytest.mark.parametrize("k", [1000, 2048])
def test_tier3_forced_large_k(k):
    """16,384 identical rows, interleaved: more than the 8192-entry tier-2 reservoir holds, so the exact brute force
    answers, ties in ascending row order."""
    base = _ln_rows(np.random.default_rng(8), 1, 768)
    P = _ln_rows(np.random.default_rng(80), 32768, 768)
    P[::2] = base
    Q = (base + 0.05 * _ln_rows(np.random.default_rng(9), 16, 768)).astype(np.float32)
    idx = _index(P)
    D, I = idx.search(Q, k)
    _same(D, I, *flat_ip_oracle.search_bruteforce(P, Q, k))
    assert (I % 2 == 0).all() and (np.diff(I, axis=1) > 0).all()
    assert idx.stats()["n_uncertified"] > 0


def test_exact_path_and_small_index_at_large_k():
    P, Q = _world()
    idx = _index(P)
    D, I = idx.search_device(torch.from_numpy(Q[:40]).cuda(), 2048, exact=True)
    Do, Io = _oracle(2048)
    _same(D.cpu().numpy(), I.cpu().numpy(), Do[:40], Io[:40])
    # fewer rows than k: faiss pads with -1 / lowest float
    Ps = _ln_rows(np.random.default_rng(11), 1200, 768)
    D, I = _index(Ps).search(Q[:9], 1500)
    _same(D, I, *flat_ip_oracle.search_bruteforce(Ps, Q[:9], 1500))
    assert (I[:, 1200:] == -1).all() and (D[:, 1200:] == np.finfo(np.float32).min).all()


def test_sharded_equals_global_at_1000():
    from ance_b200.search import merge_topk_host
    P, Q = _world()
    k, h = 1000, 30000
    qd = torch.from_numpy(Q).cuda()
    Ds, Is = [], []
    for lo, hi in ((0, h), (h, P.shape[0])):
        D, I = _index(P[lo:hi]).search_device(qd, k, row_offset=lo)
        Ds.append(D.cpu().numpy())
        Is.append(I.cpu().numpy())
    Dm, Im = merge_topk_host(Ds, Is, k)
    Dg, Ig = _index(P).search(Q, k)
    _same(Dm, Im, Dg, Ig)
    _same(Dm, Im, *_oracle(k))


def test_k_above_2048_is_refused():
    from ance_b200._lib import AnceError
    P, Q = _world()
    idx = _index(P[:5000])
    with pytest.raises(AnceError, match="2048"):
        idx.search(Q[:3], 2049)
    with pytest.raises(AnceError, match="2048"):
        idx.search_device(torch.from_numpy(Q[:3]).cuda(), 2049, exact=True)


def test_evaluate_dumps_top1000(tmp_path):
    """evaluation.evaluate_dumps at its default topN = 1000 (the notebook's cell 13) on --inference-shaped dumps."""
    from ance_b200 import evaluation as ev
    P = _ln_rows(np.random.default_rng(90), 5000, 768)
    Qd = _ln_rows(np.random.default_rng(91), 50, 768)
    p2id = np.arange(5000, dtype=np.int64)
    q2id = np.arange(50, dtype=np.int64)
    rng = np.random.default_rng(92)
    pos = {q: {int(p): 1 for p in rng.choice(5000, size=2, replace=False)} for q in range(50)}
    for r, sl in enumerate((slice(0, 2600), slice(2600, 5000))):
        np.save(tmp_path / f"passage_3__emb_p__data_obj_{r}.npy", P[sl])
        np.save(tmp_path / f"passage_3__embid_p__data_obj_{r}.npy", p2id[sl])
    np.save(tmp_path / "dev_query_3__emb_p__data_obj_0.npy", Qd)
    np.save(tmp_path / "dev_query_3__embid_p__data_obj_0.npy", q2id)
    res = ev.evaluate_dumps(str(tmp_path), 3, pos)
    _, Io = flat_ip_oracle.search(P, Qd, 1000)
    want = ev.eval_dev_query_full(q2id, p2id, pos, Io, 1000)
    assert set(res["full_rank"]) == set(want) and "recall@1000" in want
    for name, v in want.items():
        assert res["full_rank"][name] == pytest.approx(v, abs=1e-12), name


def test_marco_driver_topk_training_1000(tmp_path):
    """The refresh with --topk_training 1000 on 8000 passages (the coarse path, not the small-index brute force):
    ann_training_data_0 byte-identical to the oracle pipeline fed with the same embeddings."""
    import random
    from oracle import refresh_oracle
    from ance_b200.drivers import run_ann_data_gen as drv
    from tests.test_gpu_driver import _argv, _make_world
    data, ckpt, caches, train_pos, dev_pos, *_ = _make_world(tmp_path, n_p=8000)
    out = tmp_path / "ann"
    argv = _argv(data, ckpt, out, tmp_path) + ["--topk_training", "1000"]
    drv.main(argv)
    args = drv.get_arguments(argv)
    assert args.topk_training == 1000
    drv.set_env(args)
    _, _, model = drv.load_model(args, str(ckpt))
    be = drv.B200Backend(args, model)
    P, p2id = be.encode(str(data / "passages"), False)
    Q, q2id = be.encode(str(data / "train-query"), True)
    P, Q = P.cpu().numpy(), Q.cpu().numpy()
    assert P.shape == (8000, 768)
    idx = _index(P)
    idx.search(Q, 1000)
    assert idx.stats()["kprime"] >= 1000 and idx.stats()["n_uncertified"] < Q.shape[0]   # the coarse path ran
    _, I = flat_ip_oracle.search(P, Q, 1000)
    rng = random.Random(0)
    negs, _, _ = refresh_oracle.generate_negatives(q2id, p2id, train_pos, I, set(q2id.tolist()), 5, False, rng)
    want = "".join(refresh_oracle.training_data_lines(q2id, train_pos, negs, set(q2id.tolist()), rng))
    assert open(out / "ann_training_data_0").read() == want
