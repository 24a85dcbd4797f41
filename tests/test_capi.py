"""The C ABI: the library loads without a GPU, exports every symbol include/ance_b200.h declares, and the
host-only entry points behave.  No GPU compute is called here."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from ance_b200 import _lib
from ance_b200.search import merge_topk_host
from oracle import flat_ip_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_exported_and_bound(lib):
    hdr = open(os.path.join(ROOT, "include", "ance_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(ance_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 18
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/ance_b200.h but not exported"
    assert declared == set(_lib.SIGNATURES), "ctypes SIGNATURES and the header disagree"


def test_version_and_error_string(lib):
    assert b"sm_90a" in lib.ance_version()
    assert lib.ance_launch_count() >= 0


def test_argument_errors_do_not_need_a_gpu(lib):
    assert lib.ance_index_search(None, None, 1, 1, None, None, 0, None) == 1  # ANCE_ERR_INVALID
    assert b"null handle" in lib.ance_last_error()
    assert lib.ance_index_create(7, 10, 1, C.byref(C.c_void_p())) == 1
    assert b"multiple of 8" in lib.ance_last_error()


def test_no_cpu_fallback_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = C.c_void_p()
    assert lib.ance_index_create(64, 10, 1, C.byref(h)) == 2  # ANCE_ERR_CUDA
    from ance_b200.search import IndexFlatIP
    with pytest.raises(_lib.AnceError):
        IndexFlatIP(64)


@pytest.mark.parametrize("W,k", [(1, 5), (4, 10), (8, 200), (3, 1)])
def test_merge_topk_host_matches_oracle(W, k):
    rng = np.random.default_rng(W * 100 + k)
    n, nq, d = 777, 33, 16
    P = rng.standard_normal((n, d)).astype(np.float32)
    P[300:305] = P[0:5]  # ties across shards
    Q = rng.standard_normal((nq, d)).astype(np.float32)
    Q[0] = P[2]
    order = np.concatenate([np.arange(r, n, W) for r in range(W)])
    Pm = P[order]
    Dg, Ig = flat_ip_oracle.search_bruteforce(Pm, Q, k)
    Ds, Is, off = [], [], 0
    for r in range(W):
        m = len(range(r, n, W))
        d_, i_ = flat_ip_oracle.search_bruteforce(Pm[off:off + m], Q, k)
        Ds.append(d_)
        Is.append(np.where(i_ >= 0, i_ + off, -1))
        off += m
    Dm, Im = merge_topk_host(Ds, Is, k, n_threads=3)
    assert (Im == Ig).all() and (Dm == Dg).all()
    Do, Io = flat_ip_oracle.merge_shards(Ds, Is, k)
    assert (Im == Io).all() and (Dm == Do).all()


def test_merge_topk_host_padding_and_errors():
    D = [np.array([[3.0, 1.0, np.finfo(np.float32).min]], dtype=np.float32)]
    I = [np.array([[5, 9, -1]], dtype=np.int64)]
    Dm, Im = merge_topk_host(D + D, [I[0], I[0] + np.array([[10, 10, 0]])], 3)
    assert Im.tolist() == [[5, 15, 9]] and Dm.tolist() == [[3.0, 3.0, 1.0]]
    Dm, Im = merge_topk_host(D, I, 3)
    assert Im.tolist() == [[5, 9, -1]] and Dm[0, 2] == np.finfo(np.float32).min
    with pytest.raises(ValueError):
        merge_topk_host(D, I, 4)


def test_header_is_plain_c99_and_links_against_the_library(tmp_path):
    """include/ance_b200.h is the drop-in boundary: it must compile as C (not only C++), and a C program using it must
    link against libance_b200.so and run its host-only entry points without a GPU."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    from ance_b200 import _lib
    _lib.load()
    lib_dir = os.path.join(root, "ance_b200", "lib")
    src = tmp_path / "t.c"
    src.write_text(r'''
#include <stdio.h>
#include <string.h>
#include "ance_b200.h"
int main(void) {
  /* host-only entry points: version string, error text of a rejected call, the k-way merge */
  float d0[2] = {3.f, 1.f}, d1[2] = {2.f, 2.f}, out_d[2];
  int64_t i0[2] = {10, 11}, i1[2] = {5, 20}, out_i[2];
  const float* D[2] = {d0, d1};
  const int64_t* I[2] = {i0, i1};
  if (ance_merge_topk_host(D, I, 2, 1, 2, out_d, out_i, 1) != 0) return 1;
  if (out_i[0] != 10 || out_i[1] != 5 || out_d[1] != 2.f) return 2;   /* top-2 = (3.0, row 10), (2.0, row 5): equal scores go by the smaller row */
  if (ance_merge_topk_host(0, I, 2, 1, 2, out_d, out_i, 1) == 0) return 3;
  if (strlen(ance_last_error()) == 0) return 4;
  printf("%s\n", ance_version());
  return 0;
}
''')
    exe = tmp_path / "t"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(root, "include"),
                        str(src), "-o", str(exe), "-L", lib_dir, "-lance_b200", "-Wl,-rpath," + lib_dir],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip(), (r.returncode, r.stdout, r.stderr)


def test_varlen_tile_packing_plan(lib):
    """Host half of ance_encoder_forward_varlen: whole sequences packed into 128-row tiles (no GPU needed)."""
    import ctypes as C
    import numpy as np
    rng = np.random.default_rng(3)
    for lens, max_tokens, align in ((np.clip(rng.normal(76, 28, 3000).round(), 8, 128), 75776, 1),
                                    (np.clip(rng.normal(76, 28, 3000).round(), 8, 128), 75776, 16),
                                    (rng.integers(1, 129, 500), 4096, 1), (rng.integers(1, 129, 500), 4096, 16),
                                    (np.full(40, 128), 2048, 1), (np.ones(300), 1024, 16)):
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        B = len(lens)
        row0 = np.full(B, -1, dtype=np.int32)
        lo = np.zeros(max_tokens, dtype=np.uint8)
        hi = np.zeros(max_tokens, dtype=np.uint8)
        placed, tiles = C.c_int(), C.c_int()
        assert lib.ance_dbg_pack_varlen(lens.ctypes.data, B, max_tokens, align, row0.ctypes.data, lo.ctypes.data,
                                        hi.ctypes.data, C.byref(placed), C.byref(tiles)) == 0, lib.ance_last_error()
        n, t = placed.value, tiles.value
        assert 0 < n <= min(B, max_tokens // 16) and 0 < t <= max_tokens // 128
        owner = np.full(t * 128, -1)
        for i in range(n):
            r0, ln = int(row0[i]), int(lens[i])
            assert r0 // 128 == (r0 + ln - 1) // 128 and r0 % align == 0   # no sequence straddles a tile; slot alignment
            assert (owner[r0:r0 + ln] == -1).all()                   # no overlap
            owner[r0:r0 + ln] = i
            assert (lo[r0:r0 + ln] == r0 % 128).all() and (hi[r0:r0 + ln] == r0 % 128 + ln).all()
        free = np.where(owner == -1)[0]
        assert (lo[free] == free % 128).all() and (hi[free] == free % 128 + 1).all()   # filler rows see themselves only
        if n < B:   # the chunk ended because sequence n fits nowhere (or the sequence cap was hit)
            slot = (lens + align - 1) // align * align
            used = np.zeros(t, dtype=np.int64)
            np.add.at(used, row0[:n] // 128, slot[:n])
            assert n == max_tokens // 16 or (t == max_tokens // 128 and (128 - used).max() < slot[n])
        fill = lens[:n].sum() / (t * 128)
        if B == 3000:
            assert fill > (0.85 if align == 1 else 0.76), fill   # MARCO-like lengths: ~0.87 of the tile rows are real tokens (lengths > 64 cannot pair up)
