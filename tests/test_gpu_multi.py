"""Two-rank NCCL run of the drop-in driver (rows i % 2 per rank, all-gather of query rows, per-shard top-k,
gather + host merge) against the single-rank run of the same refresh: the output files must be byte-identical.
Skipped on boxes with fewer than two GPUs."""
import os
import subprocess
import sys

import pytest
import torch

from tests.test_gpu_driver import _argv, _make_world

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_rank_refresh_equals_single_rank(tmp_path):
    from ance_b200.drivers import run_ann_data_gen as drv
    data, ckpt, *_ = _make_world(tmp_path, n_p=3001, n_q=203, n_dev=51)
    out1, out2 = tmp_path / "ann1", tmp_path / "ann2"
    # SelectTopK mode: negatives = the first neighbours in rank order (no sampling), so they do not depend on
    # the merged query order, which differs between 1 and 2 ranks.  --varlen_align 16: a passage's embedding must not
    # depend on which passages share its attention tile (rank 0 of 2 sees every other record), else near-tied
    # neighbours may swap between the two runs.
    extra = ("--ann_measure_topk_mrr", "--varlen_align", "16")
    drv.main(_argv(data, ckpt, out1, tmp_path, extra=extra))
    env = dict(os.environ, PYTHONPATH=ROOT)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29533", "-m", "ance_b200.drivers.run_ann_data_gen",
           *_argv(data, ckpt, out2, tmp_path, extra=extra)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    # same neighbours => same negatives => same bytes (merged row order differs from the 1-rank order, so compare
    # through the files, whose ids are cache offsets)
    a = sorted(open(out1 / "ann_training_data_0").read().splitlines())
    b = sorted(open(out2 / "ann_training_data_0").read().splitlines())
    assert a == b and len(a) == 203
    import json
    assert json.load(open(out1 / "ann_ndcg_0"))["ndcg"] == pytest.approx(json.load(open(out2 / "ann_ndcg_0"))["ndcg"], abs=1e-12)
