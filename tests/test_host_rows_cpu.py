"""Host index (fp32 rows in pinned host memory): argument checks and driver flags, no GPU needed."""
import ctypes as C

import pytest

from ance_b200 import _lib


def _driver_argv(dpr):
    a = ["--data_dir", "d", "--training_dir", "t", "--init_model_dir", "i", "--model_type", "m", "--output_dir", "o",
         "--cache_dir", "c"]
    return a + (["--passage_path", "p", "--test_qa_path", "q", "--trivia_test_qa_path", "r"] if dpr else [])


@pytest.mark.parametrize("dpr", [False, True])
def test_drivers_parse_index_rows(dpr):
    from ance_b200.drivers import run_ann_data_gen as drv
    from ance_b200.drivers import run_ann_data_gen_dpr as ddrv
    parse = ddrv.get_arguments if dpr else drv.get_arguments
    assert parse(_driver_argv(dpr)).index_rows == "auto"
    for mode in ("device", "host", "auto"):
        assert parse(_driver_argv(dpr) + ["--index_rows", mode]).index_rows == mode
    with pytest.raises(SystemExit):
        parse(_driver_argv(dpr) + ["--index_rows", "disk"])


def test_create_host_argument_errors(lib):
    assert lib.ance_index_create_host(7, 10, 1, None, C.byref(C.c_void_p())) == 1   # ANCE_ERR_INVALID
    assert b"multiple of 8" in lib.ance_last_error()
    assert lib.ance_index_create_host(64, 0, 1, None, C.byref(C.c_void_p())) == 1
    assert lib.ance_index_create_host(64, 10, 1, None, None) == 1
    d, h = C.c_int64(), C.c_int64()
    assert lib.ance_index_memory(None, C.byref(d), C.byref(h)) == 1
    assert lib.ance_index_last_fetched(None) == -1


def test_host_index_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    assert lib.ance_index_create_host(64, 10, 1, None, C.byref(C.c_void_p())) == 2   # ANCE_ERR_CUDA
    from ance_b200.search import IndexFlatIP
    with pytest.raises(_lib.AnceError):
        IndexFlatIP(64, rows="host")


def test_index_rows_values_are_checked():
    import torch
    from ance_b200.search import IndexFlatIP
    with pytest.raises(ValueError):
        IndexFlatIP(64, rows="disk")
    with pytest.raises(ValueError, match="pinned"):
        IndexFlatIP(64, storage=torch.empty((10, 64)))   # an unpinned CPU tensor


def test_auto_counts_memory_cached_by_torch(monkeypatch):
    """--index_rows auto: memory torch's caching allocator holds but does not use (the previous refresh's rows) counts as
    available, so a configuration that fits on the device stays there on every refresh."""
    import argparse
    import torch
    from ance_b200.drivers import run_ann_data_gen as drv
    GiB = 2 ** 30
    n = 12_900_000   # MaxP: 6 * n * 768 + the workspace reserve = 57.7 GiB
    be = drv.B200Backend(argparse.Namespace(index_rows="auto", device=torch.device("cuda", 0)), model=None)
    state = {"free": 42 * GiB, "reserved": 37 * GiB, "allocated": 0}
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda dev=None: (state["free"], 80 * GiB))
    monkeypatch.setattr(torch.cuda, "memory_reserved", lambda dev=None: state["reserved"])
    monkeypatch.setattr(torch.cuda, "memory_allocated", lambda dev=None: state["allocated"])
    assert drv.device_memory_available(0) == 79 * GiB
    assert be.index_rows(n, 768) == "device"          # refresh 2: the old rows are cached, not in use
    state["allocated"] = 37 * GiB                      # ... unless something still holds them
    assert be.index_rows(n, 768) == "host"
    state.update(reserved=0, allocated=0, free=79 * GiB)
    assert be.index_rows(n, 768) == "device"          # refresh 1
    assert be.index_rows(21_015_324, 768) == "host"   # DPR on one 80 GB card
    for mode in ("device", "host"):
        be.args.index_rows = mode
        assert be.index_rows(n, 768) == mode
