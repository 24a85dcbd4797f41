"""The encoder at the sizes where linear() routes its act-0 GEMMs to the 128 x 256 tile (tc05_gemm_wide_kernel): QKV,
the out-projection and FFN-down of every full layer, and the training forward's FFN-up pre-activation U.  Every GEMM,
LayerNorm and attention tile of the encoder works on independent rows or sequences, so the same sequences encoded in
small batches (whose GEMMs stay below the threshold and run the 128 x 128 tile) must give bit-identical results:

  - inference: a dense pass, a query pass (two sequences per attention tile), a varlen pass (align 16) and a packed
    512-token pass, each one call of 75,776 rows, against batches of at most 32 sequences;
  - training forward: every saved activation slot of a 57,344-token call, token for token, against calls of 32
    sequences, and the four routed GEMMs of its first layer against fp64 from their own saved inputs;
  - backward: with every token of the batch a distinct id, each word-embedding gradient row is one token's gradient,
    and must equal the same row of the small calls' backwards; every parameter gradient is within the gate of fp32
    autograd through the oracle.

The tile counts of every call are asserted against the threshold computed from the device's SM count: routed calls at
or above it, small calls below.  test_gpu_gemm_wide.py::test_linear_routing_at_the_threshold shows from the kernel
names that linear() routes by that rule."""
import ctypes as C

import numpy as np
import pytest
import torch

from ance_b200 import _lib
from ance_b200.models import RobertaDot_NLL_LN, _CudaEncoder
from ance_b200.synthetic import random_roberta_state_dict, roberta_base_config
from tests import encoder_refs as ER
from tests.test_gpu_encoder_backward import _compare_grads, _oracle_loss

pytestmark = pytest.mark.gpu

FMTS = ["fp16", "bf16"]
DT16 = {"fp16": torch.float16, "bf16": torch.bfloat16}
PASS_ROWS = 75776          # one flagship encoder pass: 592 tiles of 128 rows
SMALL_ROWS = 4096          # rows of a small call: at most 32 sequences of 128 tokens
TRAIN_B, TRAIN_L = 448, 128
TRAIN_VOCAB = 60000        # more ids than the training batch has tokens: every token gets its own id


@pytest.fixture(scope="module")
def threshold():
    assert torch.cuda.is_available()
    _lib.load()
    return ER.wide_threshold(torch.cuda.get_device_properties(0).multi_processor_count)


def _assert_routed(name, rows, threshold):
    """A call of `rows` rows runs its act-0 GEMMs of N 768 and up on the wide kernel (the routing rule is pinned by
    test_gpu_gemm_wide.py::test_linear_routing_at_the_threshold)."""
    tiles = ER.wide_tiles(rows, 768)
    print(f"{name}: {rows} rows, {tiles} wide tiles at N 768 (threshold {threshold})")
    assert tiles >= threshold, (name, rows, tiles, threshold)


def _assert_small(name, rows, threshold):
    """A call of at most `rows` rows runs every GEMM (N 3072 at most) on the 128 x 128 tile."""
    assert ER.wide_tiles(rows, 3072) < threshold, (name, rows, threshold)


# ------------------------------------------------------------------------------------------------
# B. inference at routed sizes
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=FMTS)
def model12(request):
    m = RobertaDot_NLL_LN(roberta_base_config(num_hidden_layers=12))
    m.load_state_dict(random_roberta_state_dict(seed=0), strict=True)
    m.max_tokens = PASS_ROWS
    m.encoder_operand = request.param
    return m.cuda().eval(), request.param


def _synth(n, L, mean, sd, lo, seed):
    """Ragged sequences: CLS 0 first, then ids, padding 1 past the length (no row is all padding)."""
    rng = np.random.default_rng(seed)
    lens = np.clip(rng.normal(mean, sd, size=n).round(), lo, L).astype(np.int32)
    lens[:4] = [1, L, L - 1, 2]
    ids = rng.integers(3, 50265, size=(n, L)).astype(np.int32)
    ids[np.arange(L)[None, :] >= lens[:, None]] = 1
    ids[:, 0] = 0
    return ids, lens


def _routed_vs_small(name, encode, ids, lens, rows, per, threshold):
    """encode(ids, lens) of the whole batch (one call of `rows` rows) against the same sequences in batches of `per`."""
    ids_d, lens_d = torch.from_numpy(ids).cuda(), torch.from_numpy(lens).cuda()
    B, L = ids.shape
    _assert_routed(name, rows, threshold)
    _assert_small(name, per * L, threshold)
    big = encode(ids_d, lens_d, lens)
    small = torch.cat([encode(ids_d[s:s + per].contiguous(), lens_d[s:s + per].contiguous(), lens[s:s + per])
                       for s in range(0, B, per)])
    assert torch.isfinite(big).all()
    same = torch.equal(big, small)
    print(f"{name}: {B} sequences in one call == in batches of {per}: {same}")
    assert same, (name, (big - small).abs().max().item(), int((big != small).any(-1).sum()))


@torch.no_grad()
def test_dense_pass(model12, threshold):
    m, fmt = model12
    ids, lens = _synth(592, 128, 76, 28, 1, seed=1)
    _routed_vs_small(f"dense 592x128 {fmt}", lambda i, l, lh: m.encode_lens(i, l), ids, lens, 592 * 128, 32, threshold)


@torch.no_grad()
def test_query_pass(model12, threshold):
    m, fmt = model12
    ids, lens = _synth(1184, 64, 12, 8, 1, seed=2)
    _routed_vs_small(f"queries 1184x64 {fmt}", lambda i, l, lh: m.encode_lens(i, l), ids, lens, 1184 * 64, 32,
                     threshold)


def _pack_plan(lib, lens, L, align):
    """(sequences placed, tiles) of the first chunk of a packed / varlen forward on a handle of PASS_ROWS tokens."""
    B = len(lens)
    lh = torch.from_numpy(np.ascontiguousarray(lens, dtype=np.int32))
    row0 = torch.empty(B, dtype=torch.int32)
    placed, tiles = C.c_int(), C.c_int()
    if L <= 128:
        _lib.check(lib.ance_dbg_pack_varlen(lh.data_ptr(), B, PASS_ROWS, align, row0.data_ptr(), None, None,
                                            C.byref(placed), C.byref(tiles)))
    else:
        _lib.check(lib.ance_dbg_pack_packed(lh.data_ptr(), B, L, PASS_ROWS, align, row0.data_ptr(), None, None, None,
                                            C.byref(placed), C.byref(tiles)))
    return placed.value, tiles.value


@torch.no_grad()
def test_varlen_pass(model12, threshold):
    """Ragged sequences packed at align 16 into the 592 tiles of one pass (as many as the first chunk takes)."""
    m, fmt = model12
    lib = _lib.load()
    ids, lens = _synth(2000, 128, 60, 30, 1, seed=3)
    n, tiles = _pack_plan(lib, lens, 128, 16)
    ids, lens = ids[:n], lens[:n]
    assert _pack_plan(lib, lens, 128, 16) == (n, 592), (n, tiles)
    _routed_vs_small(f"varlen align 16, {n} sequences in 592 tiles {fmt}",
                     lambda i, l, lh: m.encode_lens_varlen(i, l, lens_host=torch.from_numpy(lh), align=16),
                     ids, lens, 592 * 128, 32, threshold)


@torch.no_grad()
def test_packed_512_pass(model12, threshold):
    """FirstP / MaxP-like lengths of up to 512 tokens, 148 x 512, packed at align 16 (long sequences on fresh tiles)."""
    m, fmt = model12
    lib = _lib.load()
    ids, lens = _synth(148, 512, 430, 90, 1, seed=4)
    n, tiles = _pack_plan(lib, lens, 512, 16)
    assert n == 148, n
    _routed_vs_small(f"packed 512 align 16, 148 sequences in {tiles} tiles {fmt}",
                     lambda i, l, lh: m.encode_lens_packed(i, l, lens_host=torch.from_numpy(lh), align=16),
                     ids, lens, tiles * 128, SMALL_ROWS // 512, threshold)


# ------------------------------------------------------------------------------------------------
# C / D. training at routed size: one forward_train of 448 x 128 = 57,344 tokens
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=FMTS)
def model2(request):
    fmt = request.param
    sd = random_roberta_state_dict(seed=7, n_layer=2, vocab=TRAIN_VOCAB)
    m = RobertaDot_NLL_LN(roberta_base_config(num_hidden_layers=2, vocab_size=TRAIN_VOCAB))
    m.load_state_dict(sd, strict=True)
    m.max_tokens = PASS_ROWS
    m.encoder_operand = fmt
    return m.cuda(), sd, fmt


def _train_batch(seed=11):
    """448 x 128 with ragged lengths, holed masks and a length-1 sequence; every non-padding token a distinct id (the
    first tokens included), padding id 1 past each length."""
    B, L = TRAIN_B, TRAIN_L
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[0], lens[2] = L, 1
    real = torch.arange(L)[None, :] < lens[:, None]
    mask = real & (torch.rand(B, L, generator=g) < 0.8)
    mask[:, 0] = True
    n = int(real.sum())
    assert n <= TRAIN_VOCAB - 3
    ids = torch.ones(B, L, dtype=torch.int64)
    ids[real] = 3 + torch.randperm(TRAIN_VOCAB - 3, generator=g)[:n]
    return ids, mask.to(torch.int64), real


def _slots(enc, ws, B, L, fmt):
    """The saved activations of a forward_train: {(layer, slot): [rows, cols] 16-bit}."""
    lo = (C.c_size_t * len(_lib.TRAIN_LAYOUT_FIELDS))()
    _lib.check(enc.lib.ance_dbg_train_layout(enc.h, B, L, lo))
    lo = dict(zip(_lib.TRAIN_LAYOUT_FIELDS, lo))
    M, H, F = B * L, 768, 3072
    cols = {"x_in": H, "qkv": 3 * H, "ctx": H, "t1": H, "x1": H, "u": F, "ff": F, "t2": H}
    out = {}
    for l, names in ((0, ("x_in", "qkv", "ctx", "t1", "x1", "u", "ff", "t2")), (1, ("x_in", "qkv", "ctx"))):
        base = lo["layers"] + l * lo["per_layer"]
        for s in names:
            off, n = base + lo[s], M * cols[s]
            out[(l, s)] = ws[off:off + 2 * n].view(DT16[fmt]).view(M, cols[s])
    return out


def test_forward_train_slots_and_routed_gemms(model2, threshold):
    m, _, fmt = model2
    dev = torch.device("cuda", torch.cuda.current_device())
    enc = _CudaEncoder(m.roberta, _lib.ANCE_ARCH_ROBERTA, 12, 1, (m.embeddingHead, m.norm), TRAIN_B * TRAIN_L, dev, fmt)
    ids, mask, _ = _train_batch()
    B, L = ids.shape
    i32, m8 = ids.to(torch.int32).cuda(), mask.to(torch.uint8).cuda()
    # QKV, T1, U and T2 of the full layer 0 and QKV of layer 1 route (the last layer runs the rest on the CLS rows only)
    _assert_routed(f"forward_train {B}x{L} {fmt}", B * L, threshold)
    _, ws = enc.forward_train(i32, None, m8)
    slots = _slots(enc, ws, B, L, fmt)
    per = SMALL_ROWS // L
    _assert_small("forward_train small", per * L, threshold)
    for s in range(0, B, per):
        e = min(B, s + per)
        _, ws_s = enc.forward_train(i32[s:e].contiguous(), None, m8[s:e].contiguous())
        small = _slots(enc, ws_s, e - s, L, fmt)
        for k, v in small.items():
            assert torch.equal(slots[k][s * L:e * L], v), (fmt, k, s, (slots[k][s * L:e * L].float() - v.float()).abs().max().item())
    print(f"forward_train {B}x{L} {fmt}: all 11 slots == calls of {per} sequences")
    # the four routed GEMMs of layer 0 against fp64, from the kernel's own saved inputs
    p = [t.detach() for t in _layer_params(m, 0)]
    w16 = lambda t: t.to(DT16[fmt])
    wqkv, bqkv = w16(torch.cat([p[0], p[2], p[4]])), torch.cat([p[1], p[3], p[5]])
    checks = (("QKV", slots[(0, "qkv")], slots[(0, "x_in")], wqkv, bqkv, None),
              ("T1", slots[(0, "t1")], slots[(0, "ctx")], w16(p[6]), p[7], slots[(0, "x_in")]),
              ("U", slots[(0, "u")], slots[(0, "x1")], w16(p[10]), p[11], None),
              ("T2", slots[(0, "t2")], slots[(0, "ff")], w16(p[12]), p[13], slots[(0, "x1")]))
    for name, out16, A, W, bias, R in checks:
        assert ER.wide_tiles(B * L, W.shape[0]) >= threshold
        err, rep = ER.linear_discrimination_blocked(out16, A, W, bias, R, fmt)
        print(f"forward_train layer 0 {name} {fmt}: max err / bound {err:.3f}; perturbed (fraction rejected, median "
              f"margin, rows) {rep}")
        assert err <= 1.0, (name, err)
        for k, (frac, margin, rows) in rep.items():
            assert rows >= B * L // 2 and frac == 1.0, (name, k, rep[k])
    del ws


def _layer_params(m, l):
    lay = m.roberta.encoder.layer[l]
    s, ao = lay.attention.self, lay.attention.output
    return [s.query.weight, s.query.bias, s.key.weight, s.key.bias, s.value.weight, s.value.bias, ao.dense.weight,
            ao.dense.bias, ao.LayerNorm.weight, ao.LayerNorm.bias, lay.intermediate.dense.weight,
            lay.intermediate.dense.bias, lay.output.dense.weight, lay.output.dense.bias]


def test_backward_per_token_and_oracle(model2, threshold):
    """Word-embedding gradient rows of the routed backward == those of calls of 32 sequences; every parameter gradient
    within GATE of fp32 autograd through the oracle."""
    m, sd, fmt = model2
    m.set_trainable(True)
    try:
        ids, mask, real = _train_batch()
        B, L = ids.shape
        tok = ids[real]
        assert tok.unique().numel() == tok.numel() and not bool((tok == 1).any()), "token ids must be distinct"
        w = torch.randn(B, 768, generator=torch.Generator().manual_seed(13)).cuda()
        ids_d, mask_d = ids.cuda(), mask.cuda()
        word = m.roberta.embeddings.word_embeddings.weight
        m.zero_grad(set_to_none=True)
        # forward: QKV, T1, U, T2 of layer 0, QKV of layer 1; backward: the dgrad into CTX of layer 0
        _assert_routed(f"forward_train + backward {B}x{L} {fmt}", B * L, threshold)
        (m.body_emb(ids_d, mask_d) * w).sum().backward()
        routed_word = word.grad.clone()
        # every parameter against the oracle (its autograd in slices of sequences: the objective is a sum over them)
        gref = None
        for s in range(0, B, 112):
            e = min(B, s + 112)
            _, g = _oracle_loss(sd, [(ids[s:e], mask[s:e])], lambda emb, s=s, e=e: (emb * w[s:e]).sum())
            gref = g if gref is None else {k: gref[k] + g[k] for k in gref}
            del g
        _compare_grads(m, gref, fmt, f"sum(w o emb) {B}x{L}")
        del gref
        # per token: each word row holds one token's gradient
        per = SMALL_ROWS // L
        _assert_small("backward small", per * L, threshold)
        rows_checked = 0
        for s in range(0, B, per):
            e = min(B, s + per)
            m.zero_grad(set_to_none=True)
            (m.body_emb(ids_d[s:e].contiguous(), mask_d[s:e].contiguous()) * w[s:e]).sum().backward()
            t = ids[s:e][real[s:e]].cuda()
            got, want = routed_word[t], word.grad[t]
            assert torch.equal(got, want), (fmt, s, int((got != want).any(-1).sum()), (got - want).abs().max().item())
            rows_checked += t.numel()
        assert rows_checked == int(real.sum())
        print(f"backward {B}x{L} {fmt}: {rows_checked} word-gradient rows == calls of {per} sequences")
    finally:
        m.set_trainable(False)
        m.zero_grad(set_to_none=True)
