"""Host index (ance_index_create_host / IndexFlatIP(rows="host")): the fp32 rows live in pinned host memory and the
search reads over PCIe only the candidates the pre-filter keeps.  Bit-exact (int64 labels and fp32 scores) against the
CPU oracle and identical to a device index over the same rows."""
import functools
import random

import numpy as np
import pytest
import torch

from oracle import flat_ip_oracle
from tests.test_gpu_search import _index, _ln_rows

pytestmark = pytest.mark.gpu


def _hindex(P, operand="auto", **params):
    from ance_b200.search import IndexFlatIP
    idx = IndexFlatIP(P.shape[1], capacity=max(1, P.shape[0]), operand=operand, rows="host")
    idx.add(P)
    for k, v in params.items():
        idx.set_param(k, v)
    return idx


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
@pytest.mark.parametrize("k", [1, 100, 200, 512, 1000, 2048])
def test_host_index_parity(operand, cta_group, k):
    P, Q = _world()
    idx = _hindex(P, operand, cta_group=cta_group)
    D, I = idx.search(Q, k)
    _same(D, I, *_oracle(k))
    st = idx.stats()
    assert st["nq"] == 300 and st["kprime"] >= k, st
    assert 0 < idx.last_fetched() <= st["n_candidates"]
    # the same rows in a device index: identical tensors
    qd = torch.from_numpy(Q).cuda()
    Dh, Ih = idx.search_device(qd, k)
    Dd, Id = _index(P, operand, cta_group=cta_group).search_device(qd, k)
    assert torch.equal(Dh, Dd) and torch.equal(Ih, Id)


def test_query_counts_and_whole_corpus_sweep():
    P, Q = _world()
    k = 200
    Do, Io = _oracle(k)
    idx = _hindex(P)
    for nq in (1, 7, 300):
        D, I = idx.search(Q[:nq], k)
        _same(D, I, Do[:nq], Io[:nq])
    Q2 = _ln_rows(np.random.default_rng(77), 2048, 768)
    idx2 = _hindex(P, "fp16", max_ctas=8)
    D, I = idx2.search(Q2, k)
    assert idx2.stats()["n_splits"] == 1
    _same(D, I, *flat_ip_oracle.search(P, Q2, k))


def test_prefilter_fetches_fewer_rows_than_candidates():
    """Eight row ranges of k' candidates each: the pre-filter keeps at least k per query and far fewer than all."""
    P, Q = _world()
    k = 200
    idx = _hindex(P, "fp16", n_splits=8)
    D, I = idx.search(Q, k)
    _same(D, I, *_oracle(k))
    st = idx.stats()
    assert st["n_splits"] == 8, st
    fetched = idx.last_fetched()
    assert Q.shape[0] * k <= fetched < st["n_candidates"], (fetched, st)
    print(f"fetched {fetched} of {st['n_candidates']} candidates ({fetched / st['n_candidates']:.3f})")
    # a device index fetches nothing from host memory
    dev = _index(P, "fp16", n_splits=8)
    dev.search(Q, k)
    assert dev.last_fetched() == 0


def test_tier2_and_tier3_on_host_index():
    P, Q = _world()
    k = 1000
    idx = _hindex(P, "bf16", kprime=1024, n_splits=1)
    D, I = idx.search(Q, k)
    assert idx.stats()["n_tier2"] > 0, idx.stats()
    _same(D, I, *_oracle(k))
    base = _ln_rows(np.random.default_rng(8), 1, 768)
    P3 = _ln_rows(np.random.default_rng(80), 32768, 768)
    P3[::2] = base
    Q3 = (base + 0.05 * _ln_rows(np.random.default_rng(9), 16, 768)).astype(np.float32)
    idx3 = _hindex(P3)
    D, I = idx3.search(Q3, k)
    _same(D, I, *flat_ip_oracle.search_bruteforce(P3, Q3, k))
    assert idx3.stats()["n_uncertified"] > 0


def test_exact_path_and_padding_on_host_index():
    P, Q = _world()
    idx = _hindex(P)
    D, I = idx.search_device(torch.from_numpy(Q[:40]).cuda(), 2048, exact=True)
    Do, Io = _oracle(2048)
    _same(D.cpu().numpy(), I.cpu().numpy(), Do[:40], Io[:40])
    Ps = _ln_rows(np.random.default_rng(11), 1200, 768)
    D, I = _hindex(Ps).search(Q[:9], 1500)
    _same(D, I, *flat_ip_oracle.search_bruteforce(Ps, Q[:9], 1500))
    assert (I[:, 1200:] == -1).all()


@pytest.mark.parametrize("d,n,k,params", [(256, 40000, 100, {"n_splits": 8}),          # phase A / B at d != 768
                                          (768, 40000, 100, {"n_splits": 8, "center": 0}),
                                          (768, 200, 10, {"kprime": 32})])            # n < 256: never centred
def test_other_dims_and_uncentred_rows(d, n, k, params):
    P = _ln_rows(np.random.default_rng(21), n, d)
    Q = _ln_rows(np.random.default_rng(22), 64, d)
    idx = _hindex(P, "fp16", **params)
    D, I = idx.search(Q, k)
    _same(D, I, *flat_ip_oracle.search(P, Q, k))
    st = idx.stats()
    assert 0 < idx.last_fetched() <= st["n_candidates"], st   # the host rescoring ran
    if n > 256:
        assert idx.last_fetched() < st["n_candidates"]
    Dd, Id = _index(P, "fp16", **params).search(Q, k)
    assert (Dd == D).all() and (Id == I).all()


@pytest.mark.parametrize("k", [100, 1000])
def test_brute_force_over_several_slabs(k):
    """The host index's brute force copies the rows H2D in slabs of 512 MB (174,762 rows at d = 768): 400,000 rows make
    three, with a tie across the slab boundary that must resolve to the lower global row."""
    P = _ln_rows(np.random.default_rng(31), 400000, 768)
    Q = _ln_rows(np.random.default_rng(32), 24, 768)
    P[300000] = P[5]
    Q[0] = 2 * P[5]
    idx = _hindex(P)
    D, I = idx.search_device(torch.from_numpy(Q).cuda(), k, exact=True)
    D, I = D.cpu().numpy(), I.cpu().numpy()
    _same(D, I, *flat_ip_oracle.search(P, Q, k))
    assert I[0, 0] == 5 and I[0, 1] == 300000


def test_auto_operand_rerounds_from_host_rows():
    from ance_b200 import _lib
    P = _ln_rows(np.random.default_rng(41), 20000, 768)
    Q = _ln_rows(np.random.default_rng(42), 40, 768)
    P[777] *= 1.0e4
    P[777, 0] = 1.0e5
    Do, Io = flat_ip_oracle.search_bruteforce(P, Q, 10)
    idx = _hindex(P, "auto")
    D, I = idx.search(Q, 10)
    assert idx.operand == _lib.ANCE_FMT_BF16
    assert (I == Io).all() and (D == Do).all()


def test_add_sources_agree():
    """numpy, CPU tensor, CUDA tensor (D2H) and in place into caller-owned pinned storage."""
    from ance_b200.search import IndexFlatIP
    P, Q = _world()
    P, k, n = P[:30000], 100, 30000
    res = []
    for src in ("numpy", "cpu", "cuda", "inplace"):
        if src == "inplace":
            store = torch.empty((n, 768), dtype=torch.float32, pin_memory=True)
            idx = IndexFlatIP(768, storage=store)
            assert idx.host_rows
            for s in range(0, n, 7000):
                store[s:s + 7000].copy_(torch.from_numpy(P[s:s + 7000]))
                idx.add(store[s:s + 7000])
            assert idx.memory()["host"] == 0
        else:
            idx = IndexFlatIP(768, capacity=n, rows="host")
            for s in range(0, n, 7000):
                x = P[s:s + 7000]
                idx.add(x if src == "numpy" else torch.from_numpy(x) if src == "cpu" else torch.from_numpy(x).cuda())
            assert idx.memory()["host"] == 4 * n * 768
        assert idx.ntotal == n
        res.append(idx.search(Q, k))
    Do, Io = flat_ip_oracle.search(P, Q, k)
    for D, I in res:
        _same(D, I, Do, Io)
    with pytest.raises(ValueError):
        IndexFlatIP(768, storage=torch.empty((10, 768)))   # not pinned


def test_memory_report():
    P, Q = _world()
    n, d = P.shape
    h = _hindex(P)
    h.search(Q, 2048)
    h.search(Q, 200)
    m = h.memory()
    workspace = int(2.3 * 2 ** 30)   # include/ance_b200.h: about 2.2 GB
    assert m["host"] == 4 * n * d
    assert 2 * n * d + 4 * n <= m["device"] <= 2 * n * d + 4 * n + workspace, m
    dv = _index(P)
    dv.search(Q, 200)
    assert dv.memory()["device"] >= 6 * n * d and dv.memory()["host"] == 0
    assert m["device"] < dv.memory()["device"] - 4 * n * d + workspace


def test_two_host_shards_merge_to_global():
    from ance_b200.search import merge_topk_host
    P, Q = _world()
    k, h = 1000, 30000
    qd = torch.from_numpy(Q).cuda()
    Ds, Is = [], []
    for lo, hi in ((0, h), (h, P.shape[0])):
        D, I = _hindex(P[lo:hi]).search_device(qd, k, row_offset=lo)
        Ds.append(D.cpu().numpy())
        Is.append(I.cpu().numpy())
    Dm, Im = merge_topk_host(Ds, Is, k)
    _same(Dm, Im, *_oracle(k))


def _read_all(d):
    return {p.name: p.read_bytes() for p in sorted(d.iterdir())
            if p.name.startswith(("ann_training_data_", "ann_ndcg_")) or p.name.endswith(".npy")}


def test_marco_driver_host_rows_equals_device(tmp_path):
    from ance_b200.drivers import run_ann_data_gen as drv
    from tests.test_gpu_driver import _argv, _make_world
    data, ckpt, *_ = _make_world(tmp_path, n_p=8000)
    outs = {}
    for mode in ("device", "host"):
        for extra in ((), ("--inference",)):
            out = tmp_path / f"ann_{mode}_{len(extra)}"
            random.seed(0)
            drv.main(_argv(data, ckpt, out, tmp_path, extra=("--index_rows", mode, *extra)))
            outs[mode, len(extra)] = _read_all(out)
    for inf in (0, 1):
        assert outs["device", inf] and outs["device", inf] == outs["host", inf]
    assert "ann_training_data_0" in outs["host", 0] and "ann_ndcg_0" in outs["host", 0]


def test_dpr_driver_host_rows_equals_device(tmp_path):
    from ance_b200.drivers import run_ann_data_gen as base
    from ance_b200.drivers import run_ann_data_gen_dpr as ddrv
    from tests.test_gpu_dpr import LAYERS, VOCAB, _world as dpr_world
    data, corp, ck, *_ = dpr_world(tmp_path)
    outs = {}
    for mode in ("device", "host"):
        out = tmp_path / f"ann_{mode}"
        argv = ["--data_dir", str(data), "--training_dir", str(tmp_path / "none"), "--init_model_dir", str(ck),
                "--model_type", "dpr", "--output_dir", str(out), "--cache_dir", str(tmp_path / "cache"),
                "--end_output_num", "0", "--max_seq_length", "128", "--per_gpu_eval_batch_size", "16",
                "--topk_training", "20", "--negative_sample", "5", "--passage_path", str(corp), "--test_qa_path",
                str(corp), "--trivia_test_qa_path", str(corp), "--seed", "0", "--index_rows", mode]
        args = ddrv.get_arguments(argv)
        args.num_hidden_layers, args.vocab_size = LAYERS, VOCAB
        base.set_env(args)
        random.seed(0)
        ddrv.ann_data_gen(args)
        outs[mode] = _read_all(out)
    assert "ann_training_data_0" in outs["host"] and outs["device"] == outs["host"]
