"""The rows of a packed training plan (no GPU needed; through the ance_dbg_pack_rows hook): every token (b, i) of a
sequence's planned rows sits at row0[b] + i, each exactly once, and the other rows belong to no sequence."""
import ctypes as C

import numpy as np
import pytest

from ance_b200 import _lib


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _rows(lib, lens, L, align, max_tokens):
    B = len(lens)
    lens = np.asarray(lens, np.int32)
    row0 = np.zeros(B, np.int32)
    tok = np.full(max_tokens, -7, np.int32)
    n_placed, n_tiles = C.c_int(), C.c_int()
    rc = lib.ance_dbg_pack_rows(lens.ctypes.data, B, L, max_tokens, align, row0.ctypes.data, tok.ctypes.data,
                                C.byref(n_placed), C.byref(n_tiles))
    assert rc == 0, lib.ance_last_error()
    assert n_placed.value == B
    return lens, row0, tok[:n_tiles.value * 128], n_tiles.value


@pytest.mark.parametrize("align", [1, 16])
@pytest.mark.parametrize("L", [16, 64, 100, 128, 256, 384, 512])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_row_map(lib, align, L, seed):
    rng = np.random.default_rng(seed * 1000 + L + align)
    lens = rng.integers(1, L + 1, size=24)
    lens[0], lens[-1] = L, 1
    lens, row0, tok, n_tiles = _rows(lib, lens, L, align, 1 << 15)
    assert tok.size == n_tiles * 128
    seen = np.zeros(tok.size, bool)
    for b, n in enumerate(lens):
        # the plan's rows of sequence b: its tokens, plus (long sequences, align 16) its own padding up to 32 rows
        rows = n if (align == 1 or L <= 128 or n <= 128) else min((n + 31) // 32 * 32, L)
        r = row0[b] + np.arange(rows)
        assert not seen[r].any(), b
        seen[r] = True
        np.testing.assert_array_equal(tok[r], b * L + np.arange(rows))
    assert (tok[~seen] == -1).all()
    sel = tok >= 0
    assert len(np.unique(tok[sel])) == int(sel.sum())
    if align == 16:
        assert (row0 % 16 == 0).all()


def test_rejects_bad_lengths(lib):
    row0 = np.zeros(2, np.int32)
    tok = np.zeros(1024, np.int32)
    n, t = C.c_int(), C.c_int()
    for bad in ([0, 5], [5, 65]):
        a = np.asarray(bad, np.int32)
        assert lib.ance_dbg_pack_rows(a.ctypes.data, 2, 64, 1024, 16, row0.ctypes.data, tok.ctypes.data, C.byref(n),
                                      C.byref(t)) == 1   # ANCE_ERR_INVALID
