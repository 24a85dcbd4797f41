"""Host side of searches with 512 < k <= 2048: the three CPU oracles agree bit for bit at these sizes (the GPU tests of
tests/test_gpu_search_large_k.py rely on them), and both drivers refuse an out-of-range --topk_training while parsing
arguments, before anything is encoded."""
import argparse

import numpy as np
import pytest

from oracle import flat_ip_oracle


def _rows(rng, n, d):
    x = rng.standard_normal((n, d)).astype(np.float32)
    cent = np.random.default_rng(7).standard_normal((16, d)).astype(np.float32)
    x = 0.5 * x + 0.5 * cent[rng.integers(0, 16, size=n)]
    return np.ascontiguousarray(((x - x.mean(1, keepdims=True)) / x.std(1, keepdims=True)).astype(np.float32))


@pytest.mark.parametrize("k", [1000, 2048])
@pytest.mark.parametrize("n", [6000, 1500])   # 1500 < k = 2048: -1 / lowest-float padding
def test_three_oracles_agree_at_large_k(k, n):
    rng = np.random.default_rng(k + n)
    P = _rows(rng, n, 64)
    P[n // 2:n // 2 + 300] = P[:300]                        # exact duplicates: score ties ordered by row
    Q = _rows(np.random.default_rng(3), 12, 64)
    Q[:4] = P[:4] + 0.01 * Q[:4]
    Db, Ib = flat_ip_oracle.search_bruteforce(P, Q, k)
    Ds, Is = flat_ip_oracle.search(P, Q, k)
    Dc, Ic = flat_ip_oracle.search_c(P, Q, k)
    for D, I in ((Ds, Is), (Dc, Ic)):
        assert (I == Ib).all() and (D.view(np.uint32) == Db.view(np.uint32)).all()
    kk = min(k, n)
    assert (Ib[:, kk:] == -1).all() and (Db[:, kk:] == np.finfo(np.float32).min).all()
    assert (Ib[:, :kk] >= 0).all()
    for q in range(4):                                      # the planted row and its duplicate, smaller row first
        a, b = np.where(Ib[q] == q)[0], np.where(Ib[q] == n // 2 + q)[0]
        assert len(a) == 1 and len(b) == 1 and b[0] == a[0] + 1


def _marco_args(topk):
    from ance_b200.drivers import run_ann_data_gen as drv
    return drv.get_arguments(["--data_dir", "d", "--training_dir", "t", "--init_model_dir", "i", "--model_type",
                              "rdot_nll", "--output_dir", "o", "--cache_dir", "c", "--topk_training", str(topk)])


def _dpr_args(topk):
    from ance_b200.drivers import run_ann_data_gen_dpr as ddrv
    return ddrv.get_arguments(["--data_dir", "d", "--training_dir", "t", "--init_model_dir", "i", "--model_type", "dpr",
                               "--output_dir", "o", "--cache_dir", "c", "--passage_path", "p", "--test_qa_path", "q",
                               "--trivia_test_qa_path", "r", "--topk_training", str(topk)])


@pytest.mark.parametrize("parse", [_marco_args, _dpr_args])
def test_topk_training_range_is_checked_while_parsing(parse, capsys):
    for ok in (1, 500, 1000, 2048):
        assert parse(ok).topk_training == ok
    for bad in (0, -5, 2049):
        with pytest.raises(SystemExit):
            parse(bad)
        assert "--topk_training" in capsys.readouterr().err
    from ance_b200.drivers.run_ann_data_gen import topk_arg
    with pytest.raises(argparse.ArgumentTypeError, match="2048"):
        topk_arg("4096")
