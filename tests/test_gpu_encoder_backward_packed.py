"""Packed variable-length training on the GPU: the packed training forward against the dense one (bit for bit at
varlen_align 16, with and without dropout), gradients of passage triplets, FirstP, MaxP (with all-padding chunks) and the
DPR BiEncoder under set_trainable(..., packed=True) against the oracle gate and against the dense path, rows of no sequence
carrying no gradient, the dense fallback for non-prefix masks, and the refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

from ance_b200 import _lib
from ance_b200.models import BiEncoder, RobertaDot_CLF_ANN_NLL_MultiChunk
from ance_b200.synthetic import roberta_base_config
from oracle.encoder_oracle import EncoderOracle
from tests import encoder_dropout_refs as D
from tests import encoder_grad_long_refs as R
from tests import encoder_grad_refs as G
from tests.test_gpu_encoder_backward import DT16, FMT_CODE, GATE, LOG2E, VOCAB, _batch, _compare_grads, _model, _oracle_loss
from tests.test_gpu_encoder_backward_long import _bert_oracle, _bert_sd, _maxp, _oracle_chunk

pytestmark = pytest.mark.gpu

FMTS = ["fp16", "bf16"]
# densest packing (align 1) against the dense forward: at fp16 the packed inference tests' bound (tests/test_gpu_packed.py,
# 1e-2).  Those tests run fp16 only; the bf16 bound here is that one times 8, the ratio of the two formats' unit roundoffs
# (2^-9 / 2^-12): an extrapolation, not a derived bound.
ALIGN1_ATOL = {"fp16": 1e-2, "bf16": 8e-2}
# packed (align 16) against dense gradients: the same arithmetic up to fp32 summation order in the GEMMs' row sums (the
# packed rows sit elsewhere in the tiles), measured at 2e-7 .. 5e-6 per tensor
PACKED_VS_DENSE = 1e-4


@pytest.fixture(scope="module")
def gpu_lib():
    assert torch.cuda.is_available()
    return _lib.load()


def _prefix_batch(B, L, seed, lo=1):
    """Prefix masks with lengths in [lo, L] (row 0 full), ids as _batch makes them."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(lo, L + 1, (B,), generator=g)
    lens[0] = L
    ids = torch.randint(3, VOCAB, (B, L), generator=g)
    mask = torch.arange(L)[None, :] < lens[:, None]
    ids = torch.where(mask, ids, torch.full_like(ids, 1))
    ids[:, 0] = 0
    return ids, mask.to(torch.int64)


def _grads(m):
    return {k: p.grad.detach().clone() for k, p in m.named_parameters()}


def _rel_vs(m, ref):
    """Largest per-tensor ||g - g_ref|| / ||g_ref|| of the model's gradients against another set (key biases skipped:
    their exact gradient is zero, see _compare_grads)."""
    worst = 0.0
    for k, p in m.named_parameters():
        if k.endswith("attention.self.key.bias"):
            continue
        worst = max(worst, float((p.grad - ref[k]).norm() / ref[k].norm().clamp_min(1e-30)))
    return worst


# ------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("L", [64, 128, 256, 512])
def test_packed_forward_equals_dense(gpu_lib, fmt, L):
    m, _ = _model(fmt)
    enc = m._encoder(torch.device("cuda"))
    enc.set_param("train_max_len", 512)
    ids, mask = _prefix_batch(6, L, L)
    i32 = ids.to(torch.int32).cuda()
    lens = mask.sum(1).to(torch.int32)
    for dropout in (None, (0.1, 0.1, 1234567890123)):
        ref, _ = enc.forward_train(i32, lens.cuda(), None, dropout)
        out, _ = enc.forward_train_packed(i32, lens.cuda(), lens, dropout, align=16)
        assert torch.equal(out, ref), (L, dropout)
        if dropout is None:   # densest packing: fp32 summation order inside a tile only (the packed inference bound)
            dens, _ = enc.forward_train_packed(i32, lens.cuda(), lens, None, align=1)
            assert torch.allclose(dens, ref, rtol=0, atol=ALIGN1_ATOL[fmt])
        else:                 # hidden dropout alone may run on the densest plan as well
            dens, _ = enc.forward_train_packed(i32, lens.cuda(), lens, (0.1, 0.0, 7), align=1)
            ref1, _ = enc.forward_train(i32, lens.cuda(), None, (0.1, 0.0, 7))
            assert torch.allclose(dens, ref1, rtol=0, atol=ALIGN1_ATOL[fmt])


# ------------------------------------------------------------------------------------------------
# the per-sequence attention backward (ance_dbg_attention_backward_packed)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("L", [64, 128, 256, 512])
@pytest.mark.parametrize("p_attn", [0.0, 0.1])
def test_attention_backward_per_sequence(gpu_lib, fmt, L, p_attn):
    """attn_bwd_kernel (L <= 128) and dq_kernel / dkv_kernel (above) with kSeq: sequences of random lengths (one full, one
    of 1 token, the others leaving partial 64-row blocks) placed in random order at arbitrary row offsets (gaps of 0..39
    rows, so most offsets are not multiples of 16).  Every row outside a sequence holds NaN in qkv, kbias and dout (any read
    of it would show) and must come back exactly 0; the sequences' rows are held to the dense fp64 references of
    tests/encoder_grad_refs.py / encoder_grad_long_refs.py (with dropout: encoder_dropout_refs' masked reference, its
    counters (sequence, query, key) those of the dense batch) for the same sequences padded to L."""
    g = torch.Generator().manual_seed(L * 31 + int(p_attn * 10))
    B, heads, H = 6, 3, 192
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[0], lens[1], lens[2] = L, 1, max(1, L - 37)
    keep = torch.arange(L)[None, :] < lens[:, None]
    kb = torch.where(keep, 0.0, -10000.0 * LOG2E).reshape(-1).float()
    qkv = (torch.randn(B * L, 3 * H, generator=g, dtype=torch.float64) * 1.5).to(DT16[fmt])
    order = torch.randperm(B, generator=g)
    row0 = torch.zeros(B, dtype=torch.int32)
    cur = 0
    for b in order.tolist():
        row0[b] = cur + int(torch.randint(0, 40, (1,), generator=g))
        cur = int(row0[b]) + int(lens[b])
    N = cur + int(torch.randint(1, 40, (1,), generator=g))
    inside = torch.zeros(N, dtype=torch.bool)
    src = []   # (packed rows, dense rows) of every sequence
    for b in range(B):
        r = torch.arange(int(row0[b]), int(row0[b]) + int(lens[b]))
        inside[r] = True
        src.append((r, b * L + torch.arange(int(lens[b]))))
    nan16 = torch.full((N, 3 * H), float("nan"), dtype=DT16[fmt])
    qkv_p, kb_p = nan16.clone(), torch.full((N,), float("nan"))
    for r, d in src:
        qkv_p[r], kb_p[r] = qkv[d], 0.0
    s = D.scale(p_attn) if p_attn > 0 else 1.0
    seed, layer = 0x5E9 + L, 2
    for cls_only in (0, 1):
        if cls_only:
            dout_p = torch.randn(B, H, generator=g, dtype=torch.float64).to(torch.bfloat16)
            dfull = torch.zeros(B * L, H, dtype=torch.bfloat16)
            dfull[::L] = dout_p
        else:   # padding queries have no upstream gradient (nothing reads them), as in the encoder's backward
            dfull = (torch.randn(B * L, H, generator=g, dtype=torch.float64) * keep.reshape(-1, 1)).to(torch.bfloat16)
            dout_p = torch.full((N, H), float("nan"), dtype=torch.bfloat16)
            for r, d in src:
                dout_p[r] = dfull[d]
        out = torch.full((N, 3 * H), float("nan"), device="cuda")
        dev = [t.cuda() for t in (qkv_p, kb_p, dout_p, row0, lens.to(torch.int32))]
        _lib.check(gpu_lib.ance_dbg_attention_backward_packed(
            FMT_CODE[fmt], dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(), cls_only, B, L, heads, dev[3].data_ptr(),
            dev[4].data_ptr(), N, p_attn, seed, layer, out.data_ptr(), _lib.current_stream()))
        torch.cuda.synchronize()
        out = out.cpu().double()
        assert bool((out[~inside] == 0).all()), "rows of no sequence"
        tol = G.attention_bwd_tol(qkv, kb, dfull, B, L, heads) if L <= 128 else \
            R.attention_bwd_long_tol(qkv, kb, dfull, B, L, heads, fmt)
        if p_attn > 0:
            am = torch.tensor(D.attn_masks(seed, layer, B, heads, L, p_attn))
            ref = D.masked_attention_bwd_ref(qkv, kb, dfull, B, L, heads, am, s)
            pert = D.masked_attention_bwd_ref(qkv, kb, dfull, B, L, heads, am, s, "no_mask_bwd")
            tol = tol * s * (1 + 4 * 2.0 ** -24)
        else:
            ref = G.attention_bwd_ref(qkv, kb, dfull, B, L, heads)
            pert = G.attention_bwd_ref(qkv, kb, dfull, B, L, heads, drop_jacobian=True)
        rows_p = torch.cat([r for r, _ in src])
        rows_d = torch.cat([d for _, d in src])
        err = float(((out[rows_p] - ref[rows_d]).abs() / tol[rows_d]).max())
        perr = float(((out[rows_p] - pert[rows_d]).abs() / tol[rows_d]).max())
        print(f"per-sequence attn bwd {fmt} L{L} p{p_attn} cls{cls_only}: err / bound {err:.3f}, perturbed {perr:.1f}")
        assert err <= 1.0, (L, p_attn, cls_only, err)
        assert perr > 1.0, (L, p_attn, cls_only, perr)


# ------------------------------------------------------------------------------------------------
# gradients
# ------------------------------------------------------------------------------------------------
def _passage_step(m, q, a, b, w):
    eq, ea, eb = (m.query_emb(x[0].cuda(), x[1].cuda()) for x in (q, a, b))   # three forwards, then one backward
    out = (eq * w[0]).sum() + (ea * w[1]).sum() + (eb * w[2]).sum()
    out.backward()
    return float(out)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("Ld", [128, 512])
def test_passage_triplets_packed(gpu_lib, fmt, Ld):
    """Queries of 64 tokens and passages of Ld (512: FirstP); three forwards of different length mixes before one
    backward.  Packed gradients within the oracle gate, and far closer than it to the dense path's."""
    m, sd = _model(fmt)
    q, a, b = _prefix_batch(8, 64, 81, lo=4), _prefix_batch(8, Ld, 82, lo=Ld // 8), _prefix_batch(8, Ld, 83, lo=2)
    w = torch.randn(3, 8, 768, generator=torch.Generator().manual_seed(84)).cuda()
    m.set_trainable(True, max_len=512)
    _passage_step(m, q, a, b, w)
    dense = _grads(m)
    m.zero_grad()
    m.set_trainable(True, max_len=512, packed=True)
    _passage_step(m, q, a, b, w)

    def objective(eq, ea, eb):
        return (eq * w[0]).sum() + (ea * w[1]).sum() + (eb * w[2]).sum()

    _, gref = _oracle_loss(sd, [q, a, b], objective)
    _compare_grads(m, gref, fmt, f"packed passages {Ld}")
    rel = _rel_vs(m, dense)
    print(f"packed vs dense, passages {Ld} {fmt}: worst per-tensor relative difference {rel:.2e} (gate {GATE[fmt]})")
    assert rel <= PACKED_VS_DENSE
    m.zero_grad()
    (loss,) = m(q[0].cuda(), q[1].cuda(), a[0].cuda(), a[1].cuda(), b[0].cuda(), b[1].cuda())
    m.set_trainable(True, max_len=512)
    (loss_d,) = m(q[0].cuda(), q[1].cuda(), a[0].cuda(), a[1].cuda(), b[0].cuda(), b[1].cuda())
    assert torch.equal(loss, loss_d)


@pytest.mark.parametrize("fmt", FMTS)
def test_encode_lens_packed_align1_gradients(gpu_lib, fmt):
    """The densest plan (varlen_align 1: sequences at any row, long ones across tiles) through the trainable
    encode_lens_packed: queries of 64 and passages of 512 within the oracle gate."""
    m, sd = _model(fmt)
    m.set_trainable(True, max_len=512, packed=True)
    q, a = _prefix_batch(6, 64, 121, lo=3), _prefix_batch(6, 512, 122, lo=5)
    w = torch.randn(2, 6, 768, generator=torch.Generator().manual_seed(123)).cuda()

    def enc(x):
        return m.encode_lens_packed(x[0].to(torch.int32).cuda(), x[1].sum(1).to(torch.int32).cuda(), align=1)

    out = (enc(q) * w[0]).sum() + (enc(a) * w[1]).sum()
    out.backward()

    def objective(eq, ea):
        return (eq * w[0]).sum() + (ea * w[1]).sum()

    _, gref = _oracle_loss(sd, [q, a], objective)
    _compare_grads(m, gref, fmt, "packed align 1")


@pytest.mark.parametrize("fmt", FMTS)
def test_dropout_loss_packed_equals_dense(gpu_lib, fmt):
    m, _ = _model(fmt)
    m.train()
    q, a, b = _prefix_batch(4, 64, 91, lo=4), _prefix_batch(4, 256, 92, lo=20), _prefix_batch(4, 256, 93, lo=20)
    losses, grads = [], []
    for packed in (False, True):
        m.set_trainable(True, max_len=256, dropout=0.1, packed=packed)
        m.zero_grad()
        torch.manual_seed(5)
        (loss,) = m(q[0].cuda(), q[1].cuda(), a[0].cuda(), a[1].cuda(), b[0].cuda(), b[1].cuda())
        loss.backward()
        losses.append(loss.detach())
        grads.append(_grads(m))
    assert torch.equal(losses[0], losses[1])
    rel = _rel_vs(m, grads[0])
    print(f"dropout, packed vs dense {fmt}: worst per-tensor relative difference {rel:.2e}")
    assert rel <= PACKED_VS_DENSE


@pytest.mark.parametrize("fmt", FMTS)
def test_maxp_packed_with_empty_chunks(gpu_lib, fmt):
    """test_maxp_gradients_match_the_oracle's documents under packed=True: document 1 has an all-padding chunk."""
    _, sd = _model(fmt)
    m = RobertaDot_CLF_ANN_NLL_MultiChunk(roberta_base_config(num_hidden_layers=2, vocab_size=VOCAB))
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    m.encoder_operand = fmt
    g = torch.Generator().manual_seed(51)
    ids = torch.randint(3, VOCAB, (2, 2048), generator=g)
    ids[:, ::512] = 0
    lens = torch.tensor([1700, 900])          # document 0: chunk 3 partly; document 1: chunks 2 and 3 all padding
    mask = (torch.arange(2048)[None, :] < lens[:, None]).to(torch.int64)
    ids = torch.where(mask.bool(), ids, torch.ones_like(ids))
    with torch.no_grad():
        ref_chunks = _oracle_chunk(sd, ids, mask)
    qv = (ref_chunks[1, 1] - ref_chunks[1, 0]).cuda()

    def objective(ex):
        return _maxp(ex.reshape(2, 4, 768), qv.expand(2, 768), mask.cuda()).max(-1).values.sum()

    out = []
    for packed in (False, True):
        m.set_trainable(True, max_len=512, packed=packed)
        m.zero_grad()
        emb = m.body_emb(ids.cuda(), mask.cuda())
        assert emb.shape == (2, 4, 768) and emb.grad_fn is not None
        objective(emb).backward()
        out.append((emb.detach(), _grads(m)))
    assert torch.equal(out[0][0], out[1][0])
    _, gref = _oracle_loss(sd, [(ids.reshape(8, 512), mask.reshape(8, 512))], objective)
    _compare_grads(m, gref, fmt, "packed MaxP sum of logits")
    rel = _rel_vs(m, out[0][1])
    print(f"MaxP packed vs dense {fmt}: worst per-tensor relative difference {rel:.2e}")
    assert rel <= PACKED_VS_DENSE


@pytest.mark.parametrize("fmt", FMTS)
def test_biencoder_in_batch_packed(gpu_lib, fmt):
    sd = _bert_sd(2)
    m = BiEncoder(type("A", (), {"num_hidden_layers": 2, "vocab_size": VOCAB})())
    m.load_state_dict(sd)
    m = m.cuda()
    m.encoder_operand = fmt

    def bert_batch(B, seed, lo):
        ids, mask = _prefix_batch(B, 256, seed, lo=lo)
        ids = torch.where(mask.bool(), ids, torch.zeros_like(ids))
        ids[:, 0] = 101
        return ids, mask

    q, a = bert_batch(16, 101, 4), bert_batch(16, 102, 40)
    w = torch.randn(2, 16, 768, generator=torch.Generator().manual_seed(103)).cuda() * 0.05

    def in_batch(eq, ea):
        return -torch.log_softmax(eq @ ea.T, dim=1).diagonal().mean() + (eq * w[0]).sum() + (ea * w[1]).sum()

    res = []
    for packed in (False, True):
        m.set_trainable(True, max_len=256, packed=packed)
        m.zero_grad()
        qe, ae = m(q[0].cuda(), q[1].cuda(), a[0].cuda(), a[1].cuda())
        loss = in_batch(qe, ae)
        loss.backward()
        res.append((float(loss), _grads(m)))
    assert res[0][0] == res[1][0]   # (the dense loss itself is held to the oracle by test_gpu_encoder_backward_long.py)
    _, gref = _bert_oracle(sd, q, a, None, in_batch, "in_batch")
    rel = _rel_vs(m, res[0][1])
    print(f"BiEncoder packed vs dense {fmt}: worst per-tensor relative difference {rel:.2e}")
    assert rel <= PACKED_VS_DENSE
    # the oracle gate, widened as the dense BiEncoder test widens it: the upstream gradient d loss / d embeddings comes
    # from each side's own embeddings, so add twice its measured relative error
    with torch.no_grad():
        ours = [m.query_emb(q[0].cuda(), q[1].cuda()), m.body_emb(a[0].cuda(), a[1].cuda())]
        orc = [EncoderOracle(sd, p, "bert", 2, 12, 0, 1e-12, device="cuda") for p in ("question_model.", "ctx_model.")]
        refs = [orc[0].hidden_states(q[0].cuda(), q[1].cuda())[-1][:, 0], orc[1].hidden_states(a[0].cuda(), a[1].cuda())[-1][:, 0]]
    up = []
    for es in (ours, refs):
        leaves = [e.detach().clone().requires_grad_(True) for e in es]
        in_batch(*leaves).backward()
        up.append(torch.cat([x.grad.reshape(-1) for x in leaves]))
    rel_up = float((up[0] - up[1]).norm() / up[1].norm())
    _compare_grads(m, gref, fmt, "packed BiEncoder in_batch", extra=2 * rel_up)


# ------------------------------------------------------------------------------------------------
# rows of no sequence, fallback, refusals
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [128, 512])
def test_rows_of_no_sequence_carry_no_gradient(gpu_lib, L):
    m, _ = _model("fp16")
    m.set_trainable(True, max_len=512, packed=True)
    ids, mask = _prefix_batch(5, L, 7 + L, lo=3)
    enc = m._encoder(ids.cuda().device)
    _lib.check(gpu_lib.ance_encoder_debug_grads(enc.h, -1, None, None))
    lens = mask.sum(1).to(torch.int32).numpy()
    emb = m.body_emb(ids.cuda(), mask.cuda())
    (emb * torch.randn_like(emb)).sum().backward()
    torch.cuda.synchronize()
    row0 = np.zeros(5, np.int32)
    tok = np.zeros(enc.max_tokens, np.int32)
    n_placed, n_tiles = C.c_int(), C.c_int()
    assert gpu_lib.ance_dbg_pack_rows(lens.ctypes.data, 5, L, enc.max_tokens, 16, row0.ctypes.data, tok.ctypes.data,
                                      C.byref(n_placed), C.byref(n_tiles)) == 0
    M = n_tiles.value * 128
    tok = tok[:M]
    buf = torch.empty((min(enc.max_tokens, 4096), 768), dtype=torch.float32, device="cuda")
    seen_real = False
    for slot in range(2):
        _lib.check(gpu_lib.ance_encoder_debug_grads(enc.h, slot, buf.data_ptr(), _lib.current_stream()))
        g = buf[:M].cpu()
        filler = torch.from_numpy(tok < 0)
        pad = torch.from_numpy((tok >= 0) & ((tok % L) >= lens[np.maximum(tok, 0) // L]))
        assert int(filler.sum()) + int(pad.sum()) > 0
        assert torch.count_nonzero(g[filler | pad]) == 0, slot
        seen_real |= bool(torch.count_nonzero(g[~(filler | pad)]) > 0)
    assert seen_real


@pytest.mark.parametrize("fmt", FMTS)
def test_non_prefix_mask_takes_the_dense_path(gpu_lib, fmt):
    m, _ = _model(fmt)
    ids, mask = _batch(4, 128, 111, holed=True)
    ids, mask = ids.cuda(), mask.cuda()
    w = torch.randn(4, 768, generator=torch.Generator().manual_seed(112)).cuda()
    res = []
    for packed in (False, True):
        m.set_trainable(True, packed=packed)
        m.zero_grad()
        e = m.query_emb(ids, mask)
        (e * w).sum().backward()
        res.append((e.detach(), _grads(m)))
    assert torch.equal(res[0][0], res[1][0])
    for k in res[0][1]:
        if "word_embeddings" in k or "position_embeddings" in k:   # fp32 atomics: order varies run to run
            torch.testing.assert_close(res[0][1][k], res[1][1][k], rtol=1e-5, atol=1e-6)
        else:
            assert torch.equal(res[0][1][k], res[1][1][k]), k


def test_refusals(gpu_lib):
    m, _ = _model("fp16")
    m.set_trainable(True, max_len=512, packed=True)
    enc = m._encoder(torch.device("cuda"))
    ids = torch.randint(3, VOCAB, (2, 64), dtype=torch.int32).cuda()
    for bad in ([0, 10], [10, 65]):
        lh = torch.tensor(bad, dtype=torch.int32)
        with pytest.raises(_lib.AnceError, match=r"outside \[1, 64\]"):
            enc.forward_train_packed(ids, lh.cuda(), lh)
    with pytest.raises(_lib.AnceError, match="varlen_align = 16"):
        lh = torch.tensor([10, 20], dtype=torch.int32)
        enc.forward_train_packed(ids, lh.cuda(), lh, (0.0, 0.1, 1), align=1)
    # more rows than one plan of max_tokens
    small, _ = _model("fp16")
    small.max_tokens = 1024
    small.set_trainable(True, max_len=512, packed=True)
    ids, mask = _prefix_batch(4, 512, 5, lo=400)
    with pytest.raises(_lib.AnceError, match="does not fit one plan"):
        small.body_emb(ids.cuda(), mask.cuda())
