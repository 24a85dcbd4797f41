"""ctypes binding of libance_b200.so (the C ABI declared in include/ance_b200.h).

There is no CPU fallback anywhere in this package: if the shared library is missing it is built
(nvcc cross-compiles), and if that fails, or a compute entry point is called without an sm_90
device, the call raises.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_LIB = None

ANCE_FMT_FP16 = 0
ANCE_FMT_BF16 = 1
ANCE_ERR_UNSUPPORTED = 4
ANCE_ARCH_ROBERTA = 0
ANCE_ARCH_BERT = 1


class AnceError(RuntimeError):
    pass


class SearchStats(C.Structure):
    _fields_ = [
        ("nq", C.c_int64),
        ("n_tier2", C.c_int64),
        ("n_uncertified", C.c_int64),
        ("n_candidates", C.c_int64),
        ("kprime", C.c_int32),
        ("n_splits", C.c_int32),
        ("max_eps", C.c_float),
    ]


class EncoderConfig(C.Structure):
    _fields_ = [(n, C.c_int) for n in
                ("arch", "n_layer", "hidden", "heads", "ffn", "vocab", "max_pos", "type_vocab", "pad_id")] + [
        ("ln_eps", C.c_float), ("has_head", C.c_int), ("operand_fmt", C.c_int)]


_FP = C.POINTER(C.c_float)


class LayerWeights(C.Structure):
    _fields_ = [(n, _FP) for n in
                ("q_w", "q_b", "k_w", "k_b", "v_w", "v_b", "ao_w", "ao_b", "ln1_g", "ln1_b",
                 "ff1_w", "ff1_b", "ff2_w", "ff2_b", "ln2_g", "ln2_b")]


class EncoderWeights(C.Structure):
    _fields_ = [(n, _FP) for n in ("word_emb", "pos_emb", "type_emb", "emb_ln_g", "emb_ln_b")] + [
        ("layers", C.POINTER(LayerWeights))] + [(n, _FP) for n in ("head_w", "head_b", "head_ln_g", "head_ln_b")]


class LayerGrads(C.Structure):
    """ance_layer_grads: the layout of LayerWeights, device fp32 pointers."""
    _fields_ = LayerWeights._fields_


class EncoderGrads(C.Structure):
    """ance_encoder_grads: the layout of EncoderWeights, device fp32 pointers."""
    _fields_ = [(n, _FP) for n in ("word_emb", "pos_emb", "type_emb", "emb_ln_g", "emb_ln_b")] + [
        ("layers", C.POINTER(LayerGrads))] + [(n, _FP) for n in ("head_w", "head_b", "head_ln_g", "head_ln_b")]


# name -> (restype, argtypes); also the list the "-m 'not gpu'" symbol test checks against the header
SIGNATURES = {
    "ance_version": (C.c_char_p, []),
    "ance_last_error": (C.c_char_p, []),
    "ance_launch_count": (C.c_int64, []),
    "ance_index_create": (C.c_int, [C.c_int, C.c_int64, C.c_int, C.POINTER(C.c_void_p)]),
    "ance_index_create_over": (C.c_int, [C.c_int, C.c_int64, C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]),
    "ance_index_create_host": (C.c_int, [C.c_int, C.c_int64, C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]),
    "ance_index_memory": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "ance_index_last_fetched": (C.c_int64, [C.c_void_p]),
    "ance_index_host_rows": (C.c_void_p, [C.c_void_p]),
    "ance_index_destroy": (C.c_int, [C.c_void_p]),
    "ance_index_reset": (C.c_int, [C.c_void_p]),
    "ance_index_ntotal": (C.c_int64, [C.c_void_p]),
    "ance_index_add": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "ance_index_prepare": (C.c_int, [C.c_void_p, C.c_void_p]),
    "ance_index_search": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_int64, C.c_void_p]),
    "ance_index_search_exact": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                          C.c_int64, C.c_void_p]),
    "ance_index_last_stats": (C.c_int, [C.c_void_p, C.POINTER(SearchStats)]),
    "ance_index_set_param": (C.c_int, [C.c_void_p, C.c_char_p, C.c_double]),
    "ance_merge_topk_host": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int, C.c_int64, C.c_int,
                                       C.c_void_p, C.c_void_p, C.c_int]),
    "ance_write_training_data_host": (C.c_int, [C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_int64, C.c_int, C.POINTER(C.c_int64)]),
    "ance_encoder_create": (C.c_int, [C.POINTER(EncoderConfig), C.POINTER(EncoderWeights), C.c_int,
                                      C.POINTER(C.c_void_p)]),
    "ance_encoder_destroy": (C.c_int, [C.c_void_p]),
    "ance_encoder_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                       C.c_void_p, C.c_void_p]),
    "ance_encoder_forward_varlen": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                              C.c_void_p, C.c_void_p]),
    "ance_encoder_forward_packed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                              C.c_void_p, C.c_void_p]),
    "ance_encoder_set_param": (C.c_int, [C.c_void_p, C.c_char_p, C.c_double]),
    "ance_encoder_check": (C.c_int, [C.c_void_p, C.c_void_p]),
    "ance_encoder_debug_hidden": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ance_encoder_train_workspace": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "ance_encoder_forward_train": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                             C.c_void_p, C.c_void_p, C.c_void_p]),
    "ance_encoder_forward_train_dropout": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                     C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_uint64,
                                                     C.c_void_p]),
    "ance_encoder_train_workspace_packed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "ance_encoder_forward_train_packed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                    C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_uint64, C.c_void_p]),
    "ance_encoder_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(EncoderGrads), C.c_void_p]),
    "ance_encoder_update_weights": (C.c_int, [C.c_void_p, C.POINTER(EncoderWeights), C.c_void_p]),
    "ance_encoder_debug_grads": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ance_lamb_step": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_int, C.c_void_p, C.c_void_p]),
    "ance_adamw_step": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p]),
    "ance_profile_enable": (C.c_int, [C.c_int]),
    "ance_profile_read": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_int64), C.c_int, C.c_int]),
    "ance_dbg_pack_varlen": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "ance_dbg_pack_packed": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "ance_dbg_attention_backward_packed": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                     C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_uint64,
                                                     C.c_int, C.c_void_p, C.c_void_p]),
    "ance_dbg_pack_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                     C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "ance_dbg_gemm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ance_dbg_linear": (C.c_int, [C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                  C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ance_dbg_attention": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ance_dbg_layer_norm": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                      C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "ance_dbg_attention_backward": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                              C.c_int, C.c_void_p, C.c_void_p]),
    "ance_dbg_attention_backward_long": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                   C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ance_dbg_layer_norm_backward": (C.c_int, [C.c_int, C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                               C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p]),
    "ance_dbg_gelu_backward": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "ance_dbg_embedding_backward": (C.c_int, [C.c_void_p] + [C.c_int] * 7 + [C.c_void_p] * 8),
    "ance_dbg_attention_backward_dropout": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                      C.c_int, C.c_int, C.c_float, C.c_uint64, C.c_int, C.c_void_p,
                                                      C.c_void_p]),
    "ance_dbg_dropout_bits": (C.c_int, [C.c_uint64, C.c_uint64, C.c_uint64, C.c_int64, C.c_void_p, C.c_void_p]),
    "ance_dbg_transpose_bf16": (C.c_int, [C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_int64,
                                          C.c_void_p]),
    "ance_dbg_train_layout": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "ance_dbg_train_layout_packed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_size_t),
                                               C.POINTER(C.c_int)]),
    "ance_dbg_index_state": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]),
}

# ance_dbg_index_state's items (ANCE_STATE_*), in order
INDEX_STATE_ITEMS = ("mu", "centred", "p16", "pstats", "ndelta", "q16", "qn_hat", "qn_delta", "cand_id", "cand_cnt",
                     "cand_thr", "pass", "flagged", "flagged_cnt", "flagged_thr")

# ance_dbg_train_layout's fields, in order
TRAIN_LAYOUT_FIELDS = ("ids", "kbias", "layers", "per_layer", "x_in", "qkv", "ctx", "t1", "x1", "u", "ff", "t2",
                       "x_final", "head_in", "total")
# ance_dbg_train_layout_packed's fields after TRAIN_LAYOUT_FIELDS, in order
PACKED_LAYOUT_FIELDS = ("seq_row0", "seq_len", "row_lo", "row_hi", "row_tok", "tile_kv", "cls_ctx", "cls_x", "total")


def lib_path() -> Path:
    return Path(__file__).resolve().parent / "lib" / "libance_b200.so"


def load(build_if_missing: bool = True) -> C.CDLL:
    """Load libance_b200.so, building it first when absent.  Raises if that is impossible."""
    global _LIB
    if _LIB is not None:
        return _LIB
    p = lib_path()
    if not p.exists():
        if not build_if_missing:
            raise AnceError(f"{p} is missing and there is no CPU fallback; run __graft_entry__.build()")
        from .build import build_cuda
        build_cuda()
    lib = C.CDLL(str(p))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = header / library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    _LIB = lib
    return lib


def check(status: int) -> None:
    if status != 0:
        msg = load().ance_last_error().decode("utf-8", "replace")
        raise AnceError(f"libance_b200 error {status}: {msg}")


def ptr(t) -> int:
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else t.data_ptr()


def current_stream() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream


def index_state(handle, item: str, out) -> None:
    """ance_dbg_index_state: copy `item` (one of INDEX_STATE_ITEMS) of an index handle into `out`, a contiguous torch
    tensor (CPU or CUDA) or numpy array whose size in bytes is the item's exact size (else AnceError)."""
    if hasattr(out, "data_ptr"):
        dst, nbytes = out.data_ptr(), out.numel() * out.element_size()
    else:
        dst, nbytes = out.ctypes.data, out.nbytes
    check(load().ance_dbg_index_state(handle, INDEX_STATE_ITEMS.index(item), dst, nbytes, current_stream()))


PROFILE_CLASSES = ("gemm_head", "attention", "norm_embed", "quantize", "coarse_search", "rescore", "exact",
                   "gemm_qkv", "gemm_out", "gemm_ffn1", "gemm_ffn2", "optim")


def profile_enable(on: bool = True) -> None:
    check(load().ance_profile_enable(1 if on else 0))


def profile_read(reset: bool = True) -> dict:
    """{class: (milliseconds, launches)} of device time since the last reset (synchronises)."""
    n = len(PROFILE_CLASSES)
    ms = (C.c_double * n)()
    cnt = (C.c_int64 * n)()
    check(load().ance_profile_read(ms, cnt, n, 1 if reset else 0))
    out = {PROFILE_CLASSES[i]: (ms[i], cnt[i]) for i in range(n)}
    g = [out[k] for k in ("gemm_head", "gemm_qkv", "gemm_out", "gemm_ffn1", "gemm_ffn2")]
    out["encoder_gemm"] = (sum(x[0] for x in g), sum(x[1] for x in g))
    return out
