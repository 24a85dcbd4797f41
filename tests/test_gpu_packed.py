"""ance_encoder_forward_packed: the padding-free forward for sequences of up to 512 tokens (MaxP chunks, DPR), against
the dense padded forward of the same sequences.  Exact mode (varlen_align = 16) must be bit-identical to the dense forward
at the same L; densest mode (varlen_align = 1) agrees up to fp32 summation order and stays inside the encoder gate of
tests/test_gpu_encoder.py against the fp32 oracle."""
import numpy as np
import pytest
import torch

from ance_b200.synthetic import random_roberta_state_dict, roberta_base_config
from oracle import refresh_oracle
from oracle.encoder_oracle import RobertaDotOracle

pytestmark = pytest.mark.gpu
COS, MAXABS = 0.9995, 0.03
EDGE = [1, 16, 127, 128, 129, 255, 256, 384, 511, 512]
LAYERS = 4


def _rdot(cls_name="RobertaDot_NLL_LN", max_tokens=None, n_layer=LAYERS):
    from ance_b200 import models
    m = getattr(models, cls_name)(roberta_base_config(num_hidden_layers=n_layer))
    m.load_state_dict(random_roberta_state_dict(seed=5, n_layer=n_layer), strict=True)
    if max_tokens:
        m.max_tokens = max_tokens
    return m.cuda().eval()


@pytest.fixture(scope="module")
def rdot():
    return _rdot()


def _batch(L, n, seed):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, L + 1, size=n).astype(np.int32)
    edge = [x for x in EDGE if x <= L]
    lens[:len(edge)] = edge
    lens = lens[rng.permutation(n)]
    ids = rng.integers(3, 50265, size=(n, L)).astype(np.int32)
    ids[np.arange(L)[None, :] >= lens[:, None]] = 1
    ids[:, 0] = 0
    return ids, lens


@pytest.mark.parametrize("L", [256, 512])
def test_exact_mode_is_bit_identical_to_dense(rdot, L):
    ids, lens = _batch(L, 160, L)
    ids_d, lens_d = torch.from_numpy(ids).cuda(), torch.from_numpy(lens).cuda()
    dense = rdot.encode_lens(ids_d, lens_d)
    exact = rdot.encode_lens_packed(ids_d, lens_d, lens_host=torch.from_numpy(lens), align=16)
    rdot.check_inputs()
    assert torch.isfinite(exact).all()
    assert torch.equal(exact, dense), (exact - dense).abs().max().item()
    for b in [int(np.nonzero(lens == x)[0][0]) for x in EDGE if x <= L]:   # one sequence alone
        one = rdot.encode_lens_packed(ids_d[b:b + 1].contiguous(), lens_d[b:b + 1].contiguous(), align=16)
        assert torch.equal(one[0], dense[b]), (int(lens[b]), (one[0] - dense[b]).abs().max().item())
    # a call larger than the handle's max_tokens is split into chunks; the embeddings do not change
    small = _rdot(max_tokens=2048)
    split = small.encode_lens_packed(ids_d, lens_d, align=16)
    assert torch.equal(split, dense)
    dens = small.encode_lens_packed(ids_d, lens_d, align=1)
    assert torch.allclose(dens, dense, rtol=0, atol=1e-2)


def test_densest_mode_matches_dense_and_the_oracle(rdot):
    L = 512
    ids, lens = _batch(L, 160, 7)
    ids_d, lens_d = torch.from_numpy(ids).cuda(), torch.from_numpy(lens).cuda()
    dense = rdot.encode_lens(ids_d, lens_d)
    dens = rdot.encode_lens_packed(ids_d, lens_d, align=1)
    d = (dens - dense).abs().max().item()
    assert d <= 1e-2, d
    assert torch.nn.functional.cosine_similarity(dens, dense, dim=-1).min().item() > 0.99999
    sl = slice(0, 24)
    ref = RobertaDotOracle(random_roberta_state_dict(seed=5, n_layer=LAYERS), n_layer=LAYERS, device="cuda").body_emb(
        torch.from_numpy(ids[sl]), torch.from_numpy(np.arange(L)[None, :] < lens[sl, None])).cpu()
    got = dens[sl].cpu()
    cos = torch.nn.functional.cosine_similarity(got, ref, dim=-1).min().item()
    mx = (got - ref).abs().max().item()
    assert cos >= COS and mx <= MAXABS, (cos, mx)


def test_bad_inputs(rdot):
    from ance_b200._lib import AnceError
    ones = torch.ones(2, dtype=torch.int32, device="cuda")
    with pytest.raises(AnceError):                       # L > 512
        rdot.encode_lens_packed(torch.zeros(2, 640, dtype=torch.int32, device="cuda"), ones)
    z = torch.zeros(2, 256, dtype=torch.int32, device="cuda")
    with pytest.raises(AnceError):                       # a length of 0
        rdot.encode_lens_packed(z, torch.tensor([0, 3], dtype=torch.int32, device="cuda"))
    with pytest.raises(AnceError):                       # a length above L
        rdot.encode_lens_packed(z, torch.tensor([3, 257], dtype=torch.int32, device="cuda"))


def test_multi_chunk_packed_equals_dense():
    m = _rdot("RobertaDot_CLF_ANN_NLL_MultiChunk", n_layer=2)
    rng = np.random.default_rng(9)
    dl = np.clip(rng.lognormal(np.log(1100), 0.8, size=40).round(), 20, 2048).astype(np.int32)
    dl[:6] = [1, 512, 513, 2048, 129, 1024]
    ids = np.full((40, 2048), 1, dtype=np.int32)
    for i, n in enumerate(dl):
        ids[i, :n] = rng.integers(3, 50265, size=n)
        ids[i, 0] = 0
    ids[6, 1600] = 7          # an empty chunk that is not all padding: encoded densely
    dl[6] = min(dl[6], 1024)
    ids_d, lens_d = torch.from_numpy(ids).cuda(), torch.from_numpy(dl).cuda()
    dense = m.encode_lens_multi_chunk(ids_d, lens_d)
    exact = m.encode_lens_multi_chunk_packed(ids_d, lens_d, lens_host=torch.from_numpy(dl), align=16)
    assert exact.shape == (40, 4, 768)
    assert (dl < 1537).any()                               # all-padding chunks present
    assert torch.equal(exact, dense), (exact - dense).abs().max().item()
    again = m.encode_lens_multi_chunk_packed(ids_d, lens_d, align=16)   # cached all-pad row, host lengths copied back
    assert torch.equal(again, dense)
    dens = m.encode_lens_multi_chunk_packed(ids_d, lens_d, align=1)
    assert torch.allclose(dens, dense, rtol=0, atol=1e-2)


def test_dpr_packed_equals_dense():
    from ance_b200.models import BiEncoder

    class A:
        num_hidden_layers, vocab_size = 2, 1000

    sd = {**random_roberta_state_dict(seed=1, n_layer=2, vocab=1000, max_pos=512, head=False, prefix="question_model."),
          **random_roberta_state_dict(seed=2, n_layer=2, vocab=1000, max_pos=512, head=False, prefix="ctx_model.")}
    m = BiEncoder(A())
    m.load_state_dict(sd)
    m = m.cuda().eval()
    rng = np.random.default_rng(3)
    L = 256
    lens = rng.integers(8, L + 1, size=120)
    edge = [x for x in EDGE if x <= L]
    lens[:len(edge)] = edge
    ids = np.zeros((120, L), dtype=np.int64)
    for i, n in enumerate(lens):
        ids[i, :n] = rng.integers(103, 1000, size=n)
        ids[i, 0], ids[i, n - 1] = 101, 102
    ids[11, 5] = 0            # a mask that is not a prefix: dense
    ids[12] = 0               # an empty mask: dense
    x = torch.from_numpy(ids).cuda()
    for packed, dense in ((m.body_emb_packed, m.body_emb), (m.query_emb_packed, m.query_emb)):
        want = dense(x, x != 0)
        assert torch.equal(packed(x, align=16, ids_host=torch.from_numpy(ids)), want)
        assert torch.equal(packed(x, align=16), want)
        assert torch.allclose(packed(x, align=1), want, rtol=0, atol=1e-2)
    q = x[:, :64].contiguous()                              # questions: the L <= 128 path
    assert torch.equal(m.query_emb_packed(q, align=16), m.query_emb(q, q != 0))


def _maxp_world(tmp_path):
    from transformers import RobertaConfig
    rng = np.random.default_rng(1)
    vocab, n_d = 2000, 120
    data = tmp_path / "data"
    data.mkdir()
    dlens = np.clip(rng.lognormal(6.6, 0.8, size=n_d).astype(int), 20, 2048)
    dids = np.full((n_d, 2048), 1, dtype=np.int32)
    for i, m in enumerate(dlens):
        dids[i, :m] = rng.integers(3, vocab, size=m)
        dids[i, 0] = 0
    refresh_oracle.write_cache(str(data / "passages"), dlens, dids)
    for name, n in (("train-query", 40), ("dev-query", 12)):
        lens = rng.integers(4, 20, size=n)
        ids = np.full((n, 64), 1, dtype=np.int32)
        for i, m in enumerate(lens):
            ids[i, :m] = rng.integers(3, vocab, size=m)
            ids[i, 0] = 0
        refresh_oracle.write_cache(str(data / name), lens, ids)
    with open(data / "train-qrel.tsv", "w") as f:
        for q in range(40):
            f.write(f"{q}\t{int(rng.integers(0, n_d))}\t1\n")
    with open(data / "dev-qrel.tsv", "w") as f:
        for q in range(12):
            f.write(f"{q}\t{int(rng.integers(0, n_d))}\t1\n")
    ckpt = tmp_path / "init_model"
    ckpt.mkdir()
    RobertaConfig(vocab_size=vocab, hidden_size=768, num_hidden_layers=2, num_attention_heads=12,
                  intermediate_size=3072, max_position_embeddings=514, type_vocab_size=1, layer_norm_eps=1e-5,
                  pad_token_id=1, bos_token_id=0, eos_token_id=2).save_pretrained(str(ckpt))
    torch.save(random_roberta_state_dict(seed=6, n_layer=2, vocab=vocab), str(ckpt / "pytorch_model.bin"))
    return data, ckpt


def test_maxp_refresh_is_byte_identical_with_and_without_packing(tmp_path):
    from ance_b200.drivers import run_ann_data_gen as drv
    data, ckpt = _maxp_world(tmp_path)
    outs = []
    for extra in ([], ["--no_varlen"]):
        out = tmp_path / ("ann" + "".join(extra))
        drv.main(["--data_dir", str(data), "--training_dir", str(tmp_path / "none"), "--init_model_dir", str(ckpt),
                  "--model_type", "rdot_nll_multi_chunk", "--output_dir", str(out), "--cache_dir", str(tmp_path / "c"),
                  "--end_output_num", "0", "--max_seq_length", "2048", "--max_query_length", "64",
                  "--per_gpu_eval_batch_size", "16", "--topk_training", "40", "--negative_sample", "5",
                  "--ann_chunk_factor", "1", "--reference_sampling", "--seed", "0", *extra])
        outs.append(out)
    for name in ("ann_training_data_0", "ann_ndcg_0"):
        assert (outs[0] / name).read_bytes() == (outs[1] / name).read_bytes(), name


def test_dpr_refresh_is_byte_identical_with_and_without_packing(tmp_path):
    from ance_b200.drivers import run_ann_data_gen as base
    from ance_b200.drivers import run_ann_data_gen_dpr as ddrv
    from tests.test_gpu_dpr import LAYERS as DL, VOCAB, _world
    data, corp, ck, *_ = _world(tmp_path, n_p=600, L=256)
    outs = []
    for varlen in (True, False):
        out = tmp_path / f"ann_{varlen}"
        args = ddrv.get_arguments([
            "--data_dir", str(data), "--training_dir", str(tmp_path / "none"), "--init_model_dir", str(ck),
            "--model_type", "dpr", "--output_dir", str(out), "--cache_dir", str(tmp_path / "cache"),
            "--end_output_num", "0", "--max_seq_length", "256", "--per_gpu_eval_batch_size", "16",
            "--topk_training", "20", "--negative_sample", "5", "--passage_path", str(corp), "--test_qa_path", str(corp),
            "--trivia_test_qa_path", str(corp), "--seed", "0"])
        args.num_hidden_layers, args.vocab_size = DL, VOCAB
        args.varlen = varlen          # what --no_varlen sets in the MS MARCO driver
        base.set_env(args)
        ddrv.ann_data_gen(args)
        outs.append(out)
    for name in ("ann_training_data_0", "ann_ndcg_0"):
        assert (outs[0] / name).read_bytes() == (outs[1] / name).read_bytes(), name
