"""Parity of the sm_90a encoder with (i) the golden outputs of the reference's own classes
(tests/golden/encoder_*.npz, fp32 HF eager) and (ii) the CPU oracle layer by layer.

Tolerance (floating point, stated once; BASELINE.md par. 5): weights and activations are stored in fp16
(11-bit significand) between kernels, all accumulation / LayerNorm / softmax in fp32.  Against the
reference's fp32 forward on unit-variance outputs the gate is   min cosine >= 0.9995   and
max |diff| <= 3e-2   after 12 layers, plus retrieval overlap@200 >= 0.99 against the fp32-encoded corpus
(test_retrieval_overlap_at_200).  The bf16 storage variant (8-bit significand, selectable for checkpoints
that overflow fp16) is held to max |diff| <= 0.1 (one bf16 rounding of a value in [4, 8) is already 0.0156)
and its overlap is reported next to the fp16 one."""
import os

import numpy as np
import pytest
import torch

from oracle.encoder_oracle import RobertaDotOracle, random_roberta_state_dict

pytestmark = pytest.mark.gpu
COS, MAXABS = 0.9995, 0.03
MAXABS_BF16 = 0.1


def _cfg():
    from transformers import RobertaConfig
    return RobertaConfig(vocab_size=50265, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                         intermediate_size=3072, max_position_embeddings=514, type_vocab_size=1, layer_norm_eps=1e-5,
                         pad_token_id=1, bos_token_id=0, eos_token_id=2)


def _close(a, b, maxabs=MAXABS):
    a, b = a.float().cpu(), torch.as_tensor(b).float()
    cos = torch.nn.functional.cosine_similarity(a, b, dim=-1).min().item()
    mx = (a - b).abs().max().item()
    assert cos >= COS and mx <= maxabs, f"min cosine {cos}, max abs {mx}"
    return cos, mx


@pytest.fixture(scope="module")
def rdot():
    from ance_b200.models import RobertaDot_NLL_LN
    sd = random_roberta_state_dict(seed=0)
    m = RobertaDot_NLL_LN(_cfg())
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval(), sd


def test_rdot_nll_vs_reference_golden(rdot, golden_dir):
    model, _ = rdot
    g = np.load(os.path.join(golden_dir, "encoder_rdot_nll.npz"))
    ids = torch.from_numpy(g["ids"]).cuda()
    lens = torch.from_numpy(g["lens"]).cuda()
    mask = (torch.arange(128, device="cuda")[None, :] < lens[:, None])
    emb = model.body_emb(ids.long(), mask.long())              # the reference's call signature
    assert emb.shape == (8, 768) and emb.dtype == torch.float32
    _close(emb, g["emb"])
    assert torch.equal(model.encode_lens(ids, lens), emb)       # lengths form == mask form
    qids, qlens = torch.from_numpy(g["qids"]).cuda(), torch.from_numpy(g["qlens"]).cuda()
    qmask = (torch.arange(64, device="cuda")[None, :] < qlens[:, None])
    _close(model.query_emb(qids.long(), qmask.long()), g["qemb"])  # L = 64: two sequences per attention tile


def test_layer_by_layer_vs_oracle(rdot, golden_dir):
    model, sd = rdot
    g = np.load(os.path.join(golden_dir, "encoder_rdot_nll.npz"))
    ids, lens = g["ids"], g["lens"]
    mask = np.arange(128)[None, :] < lens[:, None]
    enc = model._encoder(torch.device("cuda", torch.cuda.current_device()))
    enc.enable_debug()
    model.encode_lens(torch.from_numpy(ids).cuda(), torch.from_numpy(lens).cuda())
    hs = RobertaDotOracle(sd).enc.hidden_states(torch.from_numpy(ids), torch.from_numpy(mask))
    m = torch.from_numpy(mask.reshape(-1))
    for l in range(13):
        h = enc.hidden(l, ids.size).cpu()
        if l < 12:
            d = (h - hs[l].reshape(ids.size, -1)).abs()[m]   # real tokens; pad positions are never read downstream
        else:  # pruned last layer: the first B rows are the CLS rows (the only ones the head reads)
            h = h[:ids.shape[0]]
            d = (h - hs[l][:, 0]).abs()
        assert not torch.isnan(h).any() and d.max().item() <= MAXABS, f"layer {l}: {d.max().item()}"
    # pruning the last layer to the CLS rows does not change the embeddings
    pruned = model.encode_lens(torch.from_numpy(ids).cuda(), torch.from_numpy(lens).cuda())
    enc.set_param("prune_last_layer", 0)
    full = model.encode_lens(torch.from_numpy(ids).cuda(), torch.from_numpy(lens).cuda())
    enc.set_param("prune_last_layer", 1)
    assert torch.equal(pruned, full)


def test_ragged_batch_and_batch_invariance(rdot):
    model, _ = rdot
    rng = np.random.default_rng(3)
    ids = torch.from_numpy(rng.integers(3, 50265, size=(5, 128)).astype(np.int32)).cuda()
    ids[:, 0] = 0
    lens = torch.tensor([128, 1, 77, 128, 30], dtype=torch.int32, device="cuda")
    for b in range(5):
        ids[b, lens[b]:] = 1
    all5 = model.encode_lens(ids, lens)
    for b in range(5):  # a sequence's embedding does not depend on its batch neighbours
        one = model.encode_lens(ids[b:b + 1].contiguous(), lens[b:b + 1].contiguous())
        assert torch.equal(one[0], all5[b])
    assert torch.isfinite(all5).all()


def test_length_buckets_do_not_change_embeddings(rdot):
    model, _ = rdot
    rng = np.random.default_rng(4)
    lens = torch.tensor([1, 7, 16, 17, 31, 33, 64, 65, 100, 128, 12, 50], dtype=torch.int32, device="cuda")
    ids = torch.from_numpy(rng.integers(3, 50265, size=(12, 128)).astype(np.int32)).cuda()
    ids[:, 0] = 0
    for b in range(12):
        ids[b, lens[b]:] = 1
    dense = model.encode_lens(ids, lens)
    packed = model.encode_lens_bucketed(ids, lens)
    # same arithmetic per row; only the number of exactly-zero softmax terms differs
    assert torch.allclose(dense, packed, rtol=0, atol=2e-3)
    assert torch.nn.functional.cosine_similarity(dense, packed, dim=-1).min().item() > 0.999999


def test_multi_chunk_vs_reference_golden(golden_dir):
    from ance_b200.models import RobertaDot_CLF_ANN_NLL_MultiChunk
    sd = random_roberta_state_dict(seed=0)
    model = RobertaDot_CLF_ANN_NLL_MultiChunk(_cfg())
    model.load_state_dict(sd, strict=True)
    model = model.cuda().eval()
    g = np.load(os.path.join(golden_dir, "encoder_multi_chunk.npz"))
    ids, lens = torch.from_numpy(g["ids"]).cuda(), torch.from_numpy(g["lens"]).cuda()
    mask = (torch.arange(2048, device="cuda")[None, :] < lens[:, None])
    emb = model.body_emb(ids.long(), mask.long())
    assert emb.shape == (2, 4, 768)
    real = torch.from_numpy(g["real_chunk"])
    _close(emb.cpu()[real], g["emb"][g["real_chunk"]])
    # all-padding chunks: finite, identical to each other (the tie class of SURVEY.md §7), and equal to
    # the transformers-2.3.0 additive-mask value the oracle computes
    assert torch.isfinite(emb).all() and torch.equal(emb[1, 2], emb[1, 3])
    _close(emb[1, 2:4], np.broadcast_to(g["allpad_oracle_2_3_0"], (2, 768)).copy())
    assert torch.equal(model.encode_lens_multi_chunk(ids, lens), emb)


def test_dpr_vs_reference_golden(golden_dir):
    from ance_b200.models import BiEncoder
    g = np.load(os.path.join(golden_dir, "encoder_dpr.npz"))
    sd = {**random_roberta_state_dict(seed=int(g["seed_q"]), vocab=30522, max_pos=512, head=False,
                                      prefix="question_model."),
          **random_roberta_state_dict(seed=int(g["seed_c"]), vocab=30522, max_pos=512, head=False,
                                      prefix="ctx_model.")}
    model = BiEncoder()
    model.load_state_dict(sd)
    model = model.cuda().eval()
    ids = torch.from_numpy(g["ids"]).cuda()
    _close(model.body_emb(ids.long(), (ids != 0).long()), g["body_emb"])
    _close(model.query_emb(ids.long(), (ids != 0).long()), g["query_emb"])


def test_bad_inputs(rdot):
    from ance_b200._lib import AnceError
    model, _ = rdot
    with pytest.raises(AnceError):  # L = 100 is neither a multiple nor a divisor of 128
        model.encode_lens(torch.zeros(2, 100, dtype=torch.int32, device="cuda"),
                          torch.ones(2, dtype=torch.int32, device="cuda"))
    with pytest.raises(AnceError):
        model.query_emb(torch.zeros(1, 64, dtype=torch.long), torch.ones(1, 64, dtype=torch.long))  # CPU tensors
    # a token id outside the vocabulary: the reference's nn.Embedding raises; here the check is deferred
    ids = torch.zeros(2, 64, dtype=torch.int32, device="cuda")
    ids[1, 3] = 60000
    model.check_inputs()                       # clean so far
    model.encode_lens(ids, torch.full((2,), 8, dtype=torch.int32, device="cuda"))
    with pytest.raises(AnceError):
        model.check_inputs()
    model.check_inputs()                       # the flag is cleared once reported



def test_layer_norm_rows_per_warp_variants_are_bit_identical(rdot):
    model, _ = rdot
    g = torch.Generator(device="cuda").manual_seed(3)
    enc = model._encoder(torch.device("cuda:0"))
    ids = torch.randint(3, 50265, (300, 128), device="cuda", generator=g, dtype=torch.int32)
    lens = torch.randint(1, 129, (300,), device="cuda", generator=g, dtype=torch.int32)
    outs = []
    try:
        for r in (1, 2, 4, 3):          # 3 = two rows per warp held packed (fewer registers, more resident blocks)
            enc.set_param("ln_rows_per_warp", r)
            outs.append(model.encode_lens(ids, lens).clone())
    finally:
        enc.set_param("ln_rows_per_warp", 2)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]) and torch.equal(outs[0], outs[3])


def test_bf16_storage_variant_vs_reference_golden(golden_dir):
    """operand_fmt = bf16: same kernels, 8-bit significand storage; looser max-abs (stated at the top)."""
    from ance_b200.models import RobertaDot_NLL_LN
    m = RobertaDot_NLL_LN(_cfg())
    m.load_state_dict(random_roberta_state_dict(seed=0), strict=True)
    m.encoder_operand = "bf16"
    m = m.cuda().eval()
    g = np.load(os.path.join(golden_dir, "encoder_rdot_nll.npz"))
    emb = m.encode_lens(torch.from_numpy(g["ids"]).cuda(), torch.from_numpy(g["lens"]).cuda())
    _close(emb, g["emb"], MAXABS_BF16)
    assert m._encoder(torch.device("cuda", torch.cuda.current_device())).operand == "bf16"


def test_fp16_overflow_is_reported_not_silent():
    """A checkpoint whose activations leave the fp16 range gives inf/NaN embeddings: check_inputs() must raise and
    point at bf16, and the bf16 variant must encode the same checkpoint finitely."""
    from ance_b200._lib import AnceError
    from ance_b200.models import RobertaDot_NLL_LN
    sd = random_roberta_state_dict(seed=1, n_layer=2)
    sd["roberta.encoder.layer.0.intermediate.dense.bias"] = sd["roberta.encoder.layer.0.intermediate.dense.bias"] + 1.0e5
    cfg = _cfg()
    cfg.num_hidden_layers = 2
    ids = torch.randint(3, 50265, (4, 64), dtype=torch.int32, device="cuda")
    lens = torch.full((4,), 64, dtype=torch.int32, device="cuda")
    for operand, ok in (("fp16", False), ("bf16", True)):
        m = RobertaDot_NLL_LN(cfg)
        m.load_state_dict(sd, strict=True)
        m.encoder_operand = operand
        m = m.cuda().eval()
        emb = m.encode_lens(ids, lens)
        if ok:
            m.check_inputs()
            assert torch.isfinite(emb).all()
        else:
            with pytest.raises(AnceError, match="fp16 range"):
                m.check_inputs()


def test_retrieval_overlap_at_200(rdot):
    """BASELINE.md par. 5's second encoder gate: encode a 20,480-passage / 512-query 12-layer fixture with the sm_90a
    encoder and with the fp32 oracle, run the ORACLE search (exact fp32 inner product, top-200) on both embedding sets
    and compare the neighbour sets the trainer would consume.  The fp32 side is oracle.encoder_oracle placed on the GPU
    (plain fp32, TF32 off) and tied to its CPU run on a slice."""
    import json
    from oracle import flat_ip_oracle
    model, sd = rdot
    rng = np.random.default_rng(11)
    n_p, n_q, k = 20480, 512, 200

    def synth(n, L, mean, sdv, lo):
        lens = np.clip(rng.normal(mean, sdv, size=n).round().astype(np.int32), lo, L)
        ids = rng.integers(3, 50265, size=(n, L)).astype(np.int32)
        ids[np.arange(L)[None, :] >= lens[:, None]] = 1
        ids[:, 0] = 0
        ids[np.arange(n), lens - 1] = 2
        return ids, lens

    p_ids, p_lens = synth(n_p, 128, 76, 28, 8)
    q_ids, q_lens = synth(n_q, 64, 9, 3, 4)
    orc_gpu = RobertaDotOracle(sd, device="cuda")

    def oracle_encode(ids, lens, bs=512):
        out = []
        for s in range(0, ids.shape[0], bs):
            m = np.arange(ids.shape[1])[None, :] < lens[s:s + bs, None]
            out.append(orc_gpu.body_emb(torch.from_numpy(ids[s:s + bs]), torch.from_numpy(m)).cpu())
        return torch.cat(out).numpy()

    P_ref, Q_ref = oracle_encode(p_ids, p_lens), oracle_encode(q_ids, q_lens)
    # the GPU-placed fp32 oracle is the CPU oracle up to fp32 summation order
    cpu = RobertaDotOracle(sd).body_emb(torch.from_numpy(p_ids[:16]), torch.from_numpy(np.arange(128)[None, :] < p_lens[:16, None]))
    assert np.abs(cpu.numpy() - P_ref[:16]).max() <= 2e-4
    _, I_ref = flat_ip_oracle.search(P_ref, Q_ref, k)
    report = {"n_passages": n_p, "n_queries": n_q, "k": k}
    for operand in ("fp16", "bf16"):
        model.encoder_operand = operand
        try:
            P = model.encode_lens(torch.from_numpy(p_ids).cuda(), torch.from_numpy(p_lens).cuda()).cpu().numpy()
            Q = model.encode_lens(torch.from_numpy(q_ids).cuda(), torch.from_numpy(q_lens).cuda()).cpu().numpy()
        finally:
            model.encoder_operand = "fp16"
        _, I = flat_ip_oracle.search(P, Q, k)
        overlap = float(np.mean([len(np.intersect1d(I[i], I_ref[i])) for i in range(n_q)])) / k
        top10 = float(np.mean([len(np.intersect1d(I[i, :10], I_ref[i, :10])) for i in range(n_q)])) / 10
        cos = float((P * P_ref).sum(1).min() / 768.0)
        report[operand] = {"overlap_at_200": overlap, "overlap_at_10": top10,
                           "max_abs": float(np.abs(P - P_ref).max()), "rms": float(np.sqrt(np.mean((P - P_ref) ** 2)))}
    out_dir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    if os.path.isdir(out_dir):
        json.dump(report, open(os.path.join(out_dir, "overlap_at_200.json"), "w"), indent=1)
    print("retrieval overlap:", json.dumps(report))
    assert report["fp16"]["max_abs"] <= MAXABS, report
    assert report["fp16"]["overlap_at_200"] >= 0.99, report
    assert report["bf16"]["max_abs"] <= MAXABS_BF16, report


def test_varlen_packing_matches_dense():
    """ance_encoder_forward_varlen (whole sequences of any length packed into 128-token attention tiles, only real tokens
    computed) against the dense padded forward of the same sequences.  Not bit-identical by construction: a sequence sits at
    a different offset of its tile, which changes the grouping of the softmax row sum and the order of the P*V
    accumulation (fp32) — same bound as the bucketed path."""
    from ance_b200.models import RobertaDot_NLL_LN
    m = RobertaDot_NLL_LN(_cfg())
    m.load_state_dict(random_roberta_state_dict(seed=0), strict=True)
    m.max_tokens = 4096            # small handle: 900 sequences need several chunks of <= 32 tiles
    m = m.cuda().eval()
    rng = np.random.default_rng(21)
    lens = np.clip(rng.normal(76, 28, size=900).round(), 1, 128).astype(np.int32)
    lens[:6] = [1, 128, 127, 2, 64, 65]
    ids = rng.integers(3, 50265, size=(900, 128)).astype(np.int32)
    ids[np.arange(128)[None, :] >= lens[:, None]] = 1
    ids[:, 0] = 0
    ids_d, lens_d = torch.from_numpy(ids).cuda(), torch.from_numpy(lens).cuda()
    dense = m.encode_lens(ids_d, lens_d)
    var = m.encode_lens_varlen(ids_d, lens_d, lens_host=torch.from_numpy(lens))
    var2 = m.encode_lens_varlen(ids_d, lens_d)                       # host lengths fetched from the device copy
    m.check_inputs()
    assert torch.isfinite(var).all() and torch.equal(var, var2)
    # densest packing: same embeddings up to the fp32 summation order inside a tile (then re-rounded to fp16 12 times)
    assert torch.allclose(dense, var, rtol=0, atol=1e-2), (dense - var).abs().max().item()
    assert torch.nn.functional.cosine_similarity(dense, var, dim=-1).min().item() > 0.99999
    # ... and both sit inside the gate against the fp32 oracle (a slice, on the GPU-placed fp32 oracle)
    sl = slice(0, 96)
    ref = RobertaDotOracle(random_roberta_state_dict(seed=0), device="cuda").body_emb(
        torch.from_numpy(ids[sl]), torch.from_numpy(np.arange(128)[None, :] < lens[sl, None])).cpu()
    _close(var[sl], ref)
    _close(dense[sl], ref)
    # slots aligned to the tensor core's K step: bit-identical to the dense forward, whatever shares the tile
    al = m.encode_lens_varlen(ids_d, lens_d, align=16)
    assert torch.equal(al, dense), (al - dense).abs().max().item()
    one = m.encode_lens_varlen(ids_d[7:8].contiguous(), lens_d[7:8].contiguous(), align=16)
    assert torch.equal(one[0], dense[7])
    # queries: L = 64
    ql = lens_d[:300].clamp(max=64)
    q = m.encode_lens_varlen(ids_d[:300, :64].contiguous(), ql)
    qd = m.encode_lens(ids_d[:300, :64].contiguous(), ql)
    assert torch.allclose(q, qd, rtol=0, atol=1e-2)
    from ance_b200._lib import AnceError
    with pytest.raises(AnceError):                                   # L > 128 is the padded / bucketed path's business
        m.encode_lens_varlen(torch.zeros(2, 256, dtype=torch.int32, device="cuda"), torch.ones(2, dtype=torch.int32, device="cuda"))
