"""SURVEY.md par. 8(f) row 3, host half: the trainer's consumers of ann_training_data_N and the evaluation-only
triplet loss, pinned by fixtures produced by the reference's own functions (oracle/make_golden.py)."""
import argparse
import json
import os

import numpy as np
import pytest
import torch

from oracle import refresh_oracle


@pytest.fixture(scope="module")
def rec(golden_dir):
    return json.load(open(os.path.join(golden_dir, "trainer_records.json")))


@pytest.fixture(scope="module")
def losses(golden_dir):
    return json.load(open(os.path.join(golden_dir, "trainer_losses.json")))


def test_oracle_records_equal_reference(rec):
    a = (rec["lines"], rec["qlens"], np.asarray(rec["qids"]), rec["plens"], np.asarray(rec["pids"]), rec["Lq"], rec["Lp"])
    assert refresh_oracle.training_pairs(*a) == rec["pairs"]
    assert refresh_oracle.training_triplets(*a) == rec["triplets"]


def _caches(rec, tmp_path):
    from ance_b200.data import EmbeddingCache
    refresh_oracle.write_cache(str(tmp_path / "passages"), rec["plens"], np.asarray(rec["pids"], dtype=np.int32))
    refresh_oracle.write_cache(str(tmp_path / "train-query"), rec["qlens"], np.asarray(rec["qids"], dtype=np.int32))
    return EmbeddingCache(str(tmp_path / "train-query")), EmbeddingCache(str(tmp_path / "passages"))


def test_processing_fns_equal_reference(rec, tmp_path):
    from ance_b200.data import GetTrainingDataProcessingFn, GetTripletTrainingDataProcessingFn, StreamingDataset
    qc, pc = _caches(rec, tmp_path)
    args = argparse.Namespace(max_seq_length=rec["Lp"], max_query_length=rec["Lq"])
    with qc, pc:
        for name, mk in (("pairs", GetTrainingDataProcessingFn), ("triplets", GetTripletTrainingDataProcessingFn)):
            got = list(StreamingDataset(rec["lines"], mk(args, qc, pc)))
            assert [[t.int().tolist() if t.dim() else int(t) for t in r] for r in got] == rec[name]
            assert [str(t.dtype) for t in got[0]] == rec[name + "_dtypes"]


@pytest.mark.parametrize("world", [1, 2, 3])
def test_triplet_batch_reader_equals_stream(rec, tmp_path, world):
    from ance_b200.data import TripletBatchReader
    qc, pc = _caches(rec, tmp_path)
    with qc, pc:
        for rank in range(world):
            want = refresh_oracle.training_triplets(rec["lines"][rank::world], rec["qlens"], np.asarray(rec["qids"]),
                                                    rec["plens"], np.asarray(rec["pids"]), rec["Lq"], rec["Lp"])
            got = []
            for q, ql, p, pl, n, nl in TripletBatchReader(rec["lines"], qc, pc, 4, rec["Lq"], rec["Lp"], rank, world, pin=False):
                assert q.dtype == torch.int32 and ql.dtype == torch.int32 and q.shape[1] == rec["Lq"] and p.shape[1] == rec["Lp"]
                assert q.shape[0] <= 4
                for i in range(q.shape[0]):
                    got.append((q[i].tolist(), int(ql[i]), p[i].tolist(), int(pl[i]), n[i].tolist(), int(nl[i])))
            assert len(got) == len(want)
            for g, w in zip(got, want):   # w = ids, mask, types for query / positive / negative
                assert g[0] == w[0] and g[1] == sum(w[1]) and g[2] == w[3] and g[3] == sum(w[4]) and g[4] == w[6] and g[5] == sum(w[7])


def test_oracle_losses_equal_reference(losses, golden_dir):
    """The reference's forward() value from the reference's own embeddings of the same inputs (fp32 fixtures)."""
    g = np.load(os.path.join(golden_dir, "encoder_rdot_nll.npz"))
    q, p = g["qemb"], g["emb"]
    got = refresh_oracle.nll_triplet_loss(refresh_oracle.dot_logits(q, p[:4]), refresh_oracle.dot_logits(q, p[4:]))
    assert got == pytest.approx(losses["rdot_nll_loss"], abs=2e-4) and losses["rdot_nll_query_passthrough_ok"]
    gm = np.load(os.path.join(golden_dir, "encoder_multi_chunk.npz"))
    d, first = gm["emb"], (gm["lens"][:, None] > np.arange(4)[None, :] * 512).astype(np.float64)
    got = refresh_oracle.nll_triplet_loss(refresh_oracle.maxp_logits(q[:2], d, first),
                                          refresh_oracle.maxp_logits(q[:2], d[::-1], first[::-1]))
    assert got == pytest.approx(losses["multi_chunk_loss"], abs=2e-4)
    gd = np.load(os.path.join(golden_dir, "encoder_dpr.npz"))
    qq, cc = gd["query_emb"], gd["body_emb"]
    got = refresh_oracle.nll_triplet_loss(refresh_oracle.dot_logits(qq[:2], cc[:2]), refresh_oracle.dot_logits(qq[:2], cc[2:]))
    assert got == pytest.approx(losses["dpr_loss"], abs=2e-4)


@pytest.mark.gpu
def test_gpu_forward_loss(losses, golden_dir):
    """ance_b200 forward(): the reference's formula on the sm_90a embeddings (tight), and the reference's value
    (loose: a logit is a 768-term dot product of LayerNorm-ed vectors, |q||x| = 768, so the bf16 activation noise of
    tests/test_gpu_encoder.py -- cosine >= 0.9995 -- moves a logit by up to a few units)."""
    from transformers import RobertaConfig
    from ance_b200.models import RobertaDot_CLF_ANN_NLL_MultiChunk, RobertaDot_NLL_LN
    from oracle.encoder_oracle import random_roberta_state_dict
    cfg = RobertaConfig(vocab_size=50265, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                        intermediate_size=3072, max_position_embeddings=514, type_vocab_size=1, layer_norm_eps=1e-5,
                        pad_token_id=1, bos_token_id=0, eos_token_id=2)
    sd = random_roberta_state_dict(seed=0)
    g = np.load(os.path.join(golden_dir, "encoder_rdot_nll.npz"))
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).long().cuda()   # noqa: E731
    ids, qids = g["ids"], g["qids"]
    mask = (np.arange(128)[None, :] < g["lens"][:, None])
    qmask = (np.arange(64)[None, :] < g["qlens"][:, None])
    m = RobertaDot_NLL_LN(cfg)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    (loss,) = m(T(qids), T(qmask), T(ids[:4]), T(mask[:4]), T(ids[4:]), T(mask[4:]))
    q, p = m.query_emb(T(qids), T(qmask)).cpu().numpy(), m.body_emb(T(ids), T(mask)).cpu().numpy()
    want = refresh_oracle.nll_triplet_loss(refresh_oracle.dot_logits(q, p[:4]), refresh_oracle.dot_logits(q, p[4:]))
    assert float(loss) == pytest.approx(want, abs=1e-3)
    assert float(loss) == pytest.approx(losses["rdot_nll_loss"], abs=3.0)
    assert torch.equal(m(T(qids), T(qmask)), m.query_emb(T(qids), T(qmask)))              # is_query pass-through
    assert torch.equal(m(T(ids), T(mask), is_query=False), m.body_emb(T(ids), T(mask)))
    gm = np.load(os.path.join(golden_dir, "encoder_multi_chunk.npz"))
    dids = gm["ids"]
    dmask = (np.arange(2048)[None, :] < gm["lens"][:, None])
    mm = RobertaDot_CLF_ANN_NLL_MultiChunk(cfg)
    mm.load_state_dict(sd, strict=True)
    mm = mm.cuda().eval()
    (lossm,) = mm(T(qids[:2]), T(qmask[:2]), T(dids), T(dmask), T(dids[::-1]), T(dmask[::-1]))
    d = mm.body_emb(T(dids), T(dmask)).cpu().numpy()
    first = (gm["lens"][:, None] > np.arange(4)[None, :] * 512).astype(np.float64)
    want = refresh_oracle.nll_triplet_loss(refresh_oracle.maxp_logits(q[:2], d, first),
                                           refresh_oracle.maxp_logits(q[:2], d[::-1], first[::-1]))
    assert float(lossm) == pytest.approx(want, abs=1e-3)
    assert float(lossm) == pytest.approx(losses["multi_chunk_loss"], abs=3.0)


def test_ann_data_watcher_hot_swaps_like_the_training_loop(rec, tmp_path):
    """drivers/run_ann.py:182-228 as an object: nothing until the refresher publishes ann_ndcg_N, then the new lines
    (truncated to a multiple of the world size), the bookkeeping values the loop logs, and a reader over this rank's
    triplets; a leftover staged file or a data file without its json is never picked up."""
    from ance_b200 import postprocess
    from ance_b200.data import AnnDataWatcher
    qc, pc = _caches(rec, tmp_path)
    ann = tmp_path / "ann"
    ann.mkdir()
    lines = rec["lines"]
    with qc, pc:
        w = AnnDataWatcher(str(ann), qc, pc, 4, rec["Lq"], rec["Lp"], rank=1, world_size=2, pin=False)
        assert w.poll() is None
        (ann / "ann_training_data_0").write_text("".join(lines))          # data first ...
        open(postprocess.staging_path(str(ann / "ann_ndcg_0")), "w").write("{partial")
        assert w.poll() is None                                            # ... not visible before the json lands
        postprocess.write_ndcg(str(ann / "ann_ndcg_0"), 0.25, "out/checkpoint-3000/")
        s = w.poll()
        assert s is not None and (s.ann_no, s.dev_ndcg, s.checkpoint_no) == (0, 0.25, 3000)
        assert len(s.lines) == (len(lines) // 2) * 2 and s.ann_path.endswith("ann_training_data_0")
        want = refresh_oracle.training_triplets(s.lines[1::2], rec["qlens"], np.asarray(rec["qids"]), rec["plens"],
                                                np.asarray(rec["pids"]), rec["Lq"], rec["Lp"])
        got = sum(q.shape[0] for q, *_ in s.reader)
        assert got == len(want)
        assert w.poll() is None                                            # same refresh: no swap
        (ann / "ann_training_data_1").write_text("".join(lines[:5]))
        postprocess.write_ndcg(str(ann / "ann_ndcg_1"), 0.5, "out/checkpoint-6000/")
        s2 = w.poll()
        assert (s2.ann_no, s2.checkpoint_no, len(s2.lines)) == (1, 6000, 4) and w.poll() is None
