"""Host half of ance_encoder_forward_packed: the plan that packs whole sequences of up to 512 tokens into 128-row
attention tiles (no GPU needed; through the ance_dbg_pack_packed hook)."""
import ctypes as C

import numpy as np
import pytest

EDGE = [1, 16, 127, 128, 129, 255, 256, 384, 511, 512]


def _plan(lib, lens, L, max_tokens, align):
    lens = np.ascontiguousarray(lens, dtype=np.int32)
    B = len(lens)
    row0 = np.full(B, -1, dtype=np.int32)
    lo = np.zeros(max_tokens, dtype=np.int32)
    hi = np.zeros(max_tokens, dtype=np.int32)
    kv = np.zeros(2 * (max_tokens // 128), dtype=np.int32)
    placed, tiles = C.c_int(), C.c_int()
    rc = lib.ance_dbg_pack_packed(lens.ctypes.data, B, L, max_tokens, align, row0.ctypes.data, lo.ctypes.data,
                                  hi.ctypes.data, kv.ctypes.data, C.byref(placed), C.byref(tiles))
    assert rc == 0, lib.ance_last_error()
    n, t = placed.value, tiles.value
    return lens, n, t, row0[:n], lo[:t * 128], hi[:t * 128], kv[:2 * t].reshape(t, 2)


def _check(lens, n, t, row0, lo, hi, kv, L, max_tokens, align):
    assert 0 < n <= min(len(lens), max_tokens // 16) and 0 < t <= max_tokens // 128
    owner = np.full(t * 128, -1)
    for i in range(n):
        r0, ln = int(row0[i]), int(lens[i])
        assert (owner[r0:r0 + ln] == -1).all()                        # contiguous and disjoint
        owner[r0:r0 + ln] = i
        assert (lo[r0:r0 + ln] == r0).all() and (hi[r0:r0 + ln] == r0 + ln).all()   # own packed range
        if align == 16 and L > 128:
            if ln > 128:                                               # long: tile boundary, its own tiles
                assert r0 % 128 == 0
                pad = min((ln + 31) // 32 * 32, L)                     # its own padding rows up to the warp boundary
                assert (owner[r0 + ln:r0 + pad] == -1).all()
                owner[r0 + ln:r0 + pad] = i
                assert (lo[r0 + ln:r0 + pad] == r0).all() and (hi[r0 + ln:r0 + pad] == r0 + ln).all()
            else:
                assert r0 % 16 == 0 and r0 // 128 == (r0 + ln - 1) // 128
    free = np.where(owner == -1)[0]
    assert (lo[free] == free).all() and (hi[free] == free + 1).all()  # rows of no sequence see themselves only
    assert t * 128 <= max_tokens                                       # nothing crosses max_tokens
    for k in range(t):                                                 # a tile's keys cover every row's own range
        rows = slice(k * 128, (k + 1) * 128)
        k0, nb = kv[k]
        assert k0 == lo[rows].min() and k0 + 128 * nb >= hi[rows].max() and k0 + 128 * (nb - 1) < hi[rows].max()
        if align == 16:
            assert nb <= 4
    return owner


@pytest.mark.parametrize("align", [16, 1])
@pytest.mark.parametrize("L", [256, 512])
def test_plan_random_lengths(lib, L, align):
    rng = np.random.default_rng(L + align)
    for max_tokens in (75776, 4096, 1024):
        lens = rng.integers(1, L + 1, size=700)
        lens[:len(EDGE)] = np.minimum(EDGE, L)
        lens = lens[rng.permutation(len(lens))]
        first, total = 0, 0
        while first < len(lens):                                       # every chunk of the call
            out = _plan(lib, lens[first:], L, max_tokens, align)
            _check(*out, L, max_tokens, align)
            first += out[1]
            total += out[1]
        assert total == len(lens)


def test_plan_exact_long_sequences_are_dense_blocks(lib):
    """A long sequence's key blocks are the dense kernel's; short ones fill the free rows of its last tile."""
    lens, n, t, row0, lo, hi, kv = _plan(lib, [300, 40, 40, 200, 16], 512, 75776, 16)
    # 300 -> tiles 0-2 (320 rows); 40 -> the 64 free rows of tile 2; 40 -> tile 3; 200 -> tiles 4-5; 16 -> tile 2's last 16
    assert n == 5 and list(row0) == [0, 320, 384, 512, 368] and t == 6
    assert tuple(kv[2]) == (0, 3) and tuple(kv[3]) == (384, 1) and tuple(kv[5]) == (512, 2)


def test_plan_densest_is_contiguous(lib):
    lens, n, t, row0, lo, hi, kv = _plan(lib, [300, 40, 129, 512, 1], 512, 75776, 1)
    assert list(row0) == [0, 300, 340, 469, 981] and t == (982 + 127) // 128


def test_plan_cfg4_fill(lib):
    """MaxP chunks at the SURVEY.md cfg-4 document lengths: exact-mode rows <= 0.62 x the dense rows."""
    rng = np.random.default_rng(4)
    doc = np.clip(np.round(rng.lognormal(np.log(1100), 0.8, size=20000)), 20, 2048).astype(np.int64)
    ch = np.clip(doc[:, None] - 512 * np.arange(4)[None, :], 0, 512).reshape(-1)
    real = ch[ch > 0]
    rows = 0
    first = 0
    while first < len(real):
        _, n, t, *_ = _plan(lib, real[first:], 512, 75776, 16)
        rows += t * 128
        first += n
    dense = len(ch) * 512
    assert rows <= 0.62 * dense, rows / dense
    assert real.sum() / rows > 0.9                                     # fill: real tokens / packed rows


def test_plan_argument_errors(lib):
    row0 = np.zeros(4, dtype=np.int32)
    placed, tiles = C.c_int(), C.c_int()
    for lens, L, mt in (([0, 5], 256, 4096), ([257], 256, 4096), ([5], 513, 4096), ([300], 512, 256)):
        a = np.asarray(lens, dtype=np.int32)
        assert lib.ance_dbg_pack_packed(a.ctypes.data, len(a), L, mt, 16, row0.ctypes.data, None, None, None,
                                        C.byref(placed), C.byref(tiles)) == 1
        assert lib.ance_last_error()
