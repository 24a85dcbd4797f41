"""``--model_type`` plugin registry and the dual-encoder classes, H100-native.

Mirrors the reference's plugin surface (model/models.py:289-322):

    MSMarcoConfigDict[name] -> MSMarcoConfig{name, model_class, process_fn, use_mean, tokenizer_class, config_class}
    model = cfg.model_class.from_pretrained(path, from_tf=..., config=..., cache_dir=...)   # run_ann_data_gen.py:120-125
    model = cfg.model_class(args); model.load_state_dict(...)                              # dpr, run_ann_data_gen_dpr.py:119-124
    emb = model.query_emb(input_ids, attention_mask) / model.body_emb(...)                 # run_ann_data_gen.py:175-178

The classes are ``nn.Module``s whose parameters carry the checkpoint's own key names (SURVEY.md §8 a2),
so ``load_state_dict`` / ``.to(device)`` / DDP wrapping behave as with the reference; the forward
is NOT PyTorch: ``query_emb`` / ``body_emb`` run the hand-written sm_90a encoder of
libance_b200.so (csrc/encoder.cu).  There is no CPU path — calling them with CPU tensors raises.
Training: after ``model.set_trainable(True)`` (inputs of up to 128 tokens) or ``model.set_trainable(True, max_len=512)``
(up to 512: FirstP documents, MaxP chunks; DPR's BiEncoder needs ``max_len=256``) ``query_emb`` / ``body_emb`` /
``forward()`` build an autograd graph whose backward runs the encoder's own backward kernels, so ``loss.backward()``
fills the parameters' ``.grad``; by default the outputs carry no graph.  ``set_trainable(True, ..., dropout=True)`` adds
the reference's training-mode dropout (hidden and attention-probability rates from the config; 0.1 for DPR) while the
module is in ``train()`` mode.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import json
import os
from typing import Optional

import numpy as np
import torch
from torch import nn
from transformers import PretrainedConfig

from . import _lib


# ---------------------------------------------------------------------------------------------
# parameter skeletons with HF key names (no forward of their own)
# ---------------------------------------------------------------------------------------------
class _Holder(nn.Module):
    pass


def _linear(i, o):
    return nn.Linear(i, o)


def _backbone(vocab, hidden, n_layer, ffn, max_pos, type_vocab, pad_id, ln_eps) -> nn.Module:
    bb = _Holder()
    emb = _Holder()
    emb.word_embeddings = nn.Embedding(vocab, hidden, padding_idx=pad_id)
    emb.position_embeddings = nn.Embedding(max_pos, hidden)
    emb.token_type_embeddings = nn.Embedding(type_vocab, hidden)
    emb.LayerNorm = nn.LayerNorm(hidden, eps=ln_eps)
    bb.embeddings = emb
    enc = _Holder()
    layers = []
    for _ in range(n_layer):
        l = _Holder()
        att = _Holder()
        slf = _Holder()
        slf.query, slf.key, slf.value = _linear(hidden, hidden), _linear(hidden, hidden), _linear(hidden, hidden)
        att.self = slf
        ao = _Holder()
        ao.dense = _linear(hidden, hidden)
        ao.LayerNorm = nn.LayerNorm(hidden, eps=ln_eps)
        att.output = ao
        l.attention = att
        inter = _Holder()
        inter.dense = _linear(hidden, ffn)
        l.intermediate = inter
        outp = _Holder()
        outp.dense = _linear(ffn, hidden)
        outp.LayerNorm = nn.LayerNorm(hidden, eps=ln_eps)
        l.output = outp
        layers.append(l)
    enc.layer = nn.ModuleList(layers)
    bb.encoder = enc
    return bb


def _np(t: torch.Tensor) -> np.ndarray:
    return np.ascontiguousarray(t.detach().float().cpu().numpy())


_EMB_FIELDS = ("word_emb", "pos_emb", "type_emb", "emb_ln_g", "emb_ln_b")
_HEAD_FIELDS = ("head_w", "head_b", "head_ln_g", "head_ln_b")


def _param_groups(backbone: nn.Module, head: Optional[tuple]):
    """The parameters in the order of ance_encoder_weights: embeddings (5), per layer the 16 of ance_layer_weights, head
    (4, or none)."""
    if hasattr(backbone, "kernel_params"):   # a backbone under other names (SEED-Encoder) lists its own
        embs, layers = backbone.kernel_params()
        hd = [] if head is None else [head[0].weight, head[0].bias, head[1].weight, head[1].bias]
        return embs, layers, hd
    emb = backbone.embeddings
    embs = [emb.word_embeddings.weight, emb.position_embeddings.weight, emb.token_type_embeddings.weight,
            emb.LayerNorm.weight, emb.LayerNorm.bias]
    layers = []
    for l in backbone.encoder.layer:
        s, ao = l.attention.self, l.attention.output
        layers.append([s.query.weight, s.query.bias, s.key.weight, s.key.bias, s.value.weight, s.value.bias,
                       ao.dense.weight, ao.dense.bias, ao.LayerNorm.weight, ao.LayerNorm.bias,
                       l.intermediate.dense.weight, l.intermediate.dense.bias,
                       l.output.dense.weight, l.output.dense.bias, l.output.LayerNorm.weight, l.output.LayerNorm.bias])
    hd = [] if head is None else [head[0].weight, head[0].bias, head[1].weight, head[1].bias]
    return embs, layers, hd


def _fill(struct_cls, layer_cls, groups, ptr):
    """ctypes weight / gradient struct over `groups` (see _param_groups); ptr maps a tensor to a float pointer.  Returns
    (struct, layer array): both must stay alive until the call that reads them returns."""
    embs, layers, hd = groups
    lw = (layer_cls * len(layers))()
    for i, ts in enumerate(layers):
        for (name, _), t in zip(layer_cls._fields_, ts):
            setattr(lw[i], name, ptr(t))
    w = struct_cls()
    for name, t in zip(_EMB_FIELDS, embs):
        setattr(w, name, ptr(t))
    w.layers = lw
    for name, t in zip(_HEAD_FIELDS, hd):
        setattr(w, name, ptr(t))
    return w, lw


def _load_checkpoint(model: nn.Module, path: str) -> nn.Module:
    """Load `path`'s pytorch_model.bin / model.safetensors into `model` and put it in eval() mode: tensors the model does
    not have are ignored, a tensor it has that the checkpoint lacks raises KeyError."""
    sd = None
    for fn in ("pytorch_model.bin", "model.safetensors"):
        p = os.path.join(path, fn)
        if os.path.exists(p):
            if fn.endswith(".bin"):
                sd = torch.load(p, map_location="cpu", weights_only=True)
            else:
                from safetensors.torch import load_file
                sd = load_file(p)
            break
    if sd is None:
        raise FileNotFoundError(f"no pytorch_model.bin / model.safetensors under {path}")
    own = model.state_dict()
    missing = [k for k in own if k not in sd]
    if missing:
        raise KeyError(f"checkpoint {path} lacks {len(missing)} tensors, e.g. {missing[:3]}")
    model.load_state_dict({k: sd[k] for k in own}, strict=True)
    model.eval()
    return model


def _dev_ptr(t: torch.Tensor):
    return C.cast(C.c_void_p(t.data_ptr()), C.POINTER(C.c_float))


class _CudaEncoder:
    """Owns one ance_encoder handle built from a backbone's current parameters."""

    def __init__(self, backbone: nn.Module, arch: int, heads: int, pad_id: int, head: Optional[tuple],
                 max_tokens: int, device: torch.device, operand: str = "fp16"):
        lib = _lib.load()
        self.lib = lib
        self.device = device
        groups = _param_groups(backbone, head)
        embs, layers, _ = groups
        H = embs[0].shape[1]
        cfg = _lib.EncoderConfig()
        cfg.arch = arch
        cfg.n_layer = len(layers)
        cfg.hidden = H
        cfg.heads = heads
        cfg.ffn = layers[0][10].shape[0]   # ff1_w [ffn, hidden]
        cfg.vocab = embs[0].shape[0]
        cfg.max_pos = embs[1].shape[0]
        cfg.type_vocab = embs[2].shape[0]
        cfg.pad_id = pad_id
        cfg.ln_eps = float(backbone.ln_eps if hasattr(backbone, "kernel_params") else backbone.embeddings.LayerNorm.eps)
        cfg.has_head = 1 if head is not None else 0
        cfg.operand_fmt = {"fp16": _lib.ANCE_FMT_FP16, "bf16": _lib.ANCE_FMT_BF16}[operand]
        self.operand = operand
        keep = []  # host arrays must outlive the create call

        def fp(t):
            a = _np(t)
            keep.append(a)
            return a.ctypes.data_as(C.POINTER(C.c_float))

        if head is not None:
            lin, norm = head
            if tuple(lin.weight.shape) != (H, H) or tuple(norm.weight.shape) != (H,):
                # ance_encoder_create reads a hidden x hidden head: any other shape would be read out of bounds
                raise _lib.AnceError(f"the CUDA encoder's head must be Linear({H}, {H}) + LayerNorm({H}), got "
                                     f"weight {tuple(lin.weight.shape)}")
        w, lw = _fill(_lib.EncoderWeights, _lib.LayerWeights, groups, fp)
        self.hidden_size = H
        self.pad_id = int(pad_id)
        self.max_tokens = int(max_tokens)
        h = C.c_void_p()
        with torch.cuda.device(device):
            _lib.check(lib.ance_encoder_create(C.byref(cfg), C.byref(w), self.max_tokens, C.byref(h)))
        self.h = h

    def __del__(self):
        try:
            if getattr(self, "h", None) is not None:
                self.lib.ance_encoder_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def set_param(self, name: str, value: float):
        _lib.check(self.lib.ance_encoder_set_param(self.h, name.encode(), float(value)))

    def check(self):
        """Raise if any forward since the last check saw an out-of-range token id / position (synchronises)."""
        with torch.cuda.device(self.device):
            _lib.check(self.lib.ance_encoder_check(self.h, C.c_void_p(torch.cuda.current_stream().cuda_stream)))

    def enable_debug(self):
        """Capture hidden states of batches up to 4096 tokens (parity tests only)."""
        _lib.check(self.lib.ance_encoder_debug_hidden(self.h, -1, None, None))

    def hidden(self, layer: int, n_tokens: int) -> torch.Tensor:
        """Hidden states after `layer` (0 = embeddings) of the last forward, fp32 [n_tokens, H]."""
        buf = torch.empty((min(self.max_tokens, 4096), self.hidden_size), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.ance_encoder_debug_hidden(self.h, layer, buf.data_ptr(), _lib.current_stream()))
        return buf[:n_tokens]

    def forward(self, ids: torch.Tensor, lens: Optional[torch.Tensor], mask: Optional[torch.Tensor],
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """ids int32 [B, L] CUDA; exactly one of lens int32 [B] / mask uint8 [B, L].  -> fp32 [B, H] (written into `out`
        when given: a contiguous fp32 CUDA tensor [B, H], e.g. a slice of an index's row storage)."""
        B, L = ids.shape
        if out is None:
            out = torch.empty((B, self.hidden_size), dtype=torch.float32, device=ids.device)
        elif out.shape != (B, self.hidden_size) or out.dtype != torch.float32 or not out.is_contiguous() or out.device != ids.device:
            raise ValueError("out must be a contiguous float32 tensor [B, hidden] on the inputs' device")
        per = max(1, min(self.max_tokens // L, self.max_tokens // 16))
        with torch.cuda.device(ids.device):
            st = _lib.current_stream()
            for s in range(0, B, per):
                e = min(B, s + per)
                _lib.check(self.lib.ance_encoder_forward(
                    self.h, ids[s:e].data_ptr(), None if lens is None else lens[s:e].data_ptr(),
                    None if mask is None else mask[s:e].data_ptr(), e - s, L, out[s:e].data_ptr(), st))
        return out

    def update_weights(self, backbone: nn.Module, head: Optional[tuple]) -> bool:
        """Refresh the handle in place from the parameters' current values (device fp32, no host round trip); False
        when a parameter is not a contiguous fp32 tensor on this encoder's device (the caller then rebuilds)."""
        groups = _param_groups(backbone, head)
        flat = groups[0] + [t for l in groups[1] for t in l] + groups[2]
        key = tuple(t.data_ptr() for t in flat)
        cached = self.__dict__.get("_weights_dev")
        if cached is None or cached[0] != key:   # the pointer struct is rebuilt only when a parameter's storage moved
            dev = self.device.index if self.device.index is not None else torch.cuda.current_device()
            if any(not t.is_cuda or t.get_device() != dev or t.dtype != torch.float32 or not t.is_contiguous() for t in flat):
                return False
            cached = self._weights_dev = (key,) + _fill(_lib.EncoderWeights, _lib.LayerWeights, groups, _dev_ptr)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.ance_encoder_update_weights(self.h, C.byref(cached[1]), _lib.current_stream()))
        self.__dict__.pop("_allpad", None)   # values cached per weights
        return True

    def forward_train(self, ids: torch.Tensor, lens: Optional[torch.Tensor], mask: Optional[torch.Tensor],
                      dropout: Optional[tuple] = None):
        """forward() of a whole [B, L] batch (L <= 128, or a multiple of 128 up to the handle's train_max_len) that also
        keeps what the backward needs; dropout = (p_hidden, p_attn, seed) runs it in training mode
        (ance_encoder_forward_train_dropout).  -> (out fp32 [B, H], workspace tensor for backward())."""
        B, L = ids.shape
        n = C.c_size_t()
        _lib.check(self.lib.ance_encoder_train_workspace(self.h, B, L, C.byref(n)))
        ws = torch.empty(n.value, dtype=torch.uint8, device=ids.device)
        out = torch.empty((B, self.hidden_size), dtype=torch.float32, device=ids.device)
        args = (self.h, ids.data_ptr(), None if lens is None else lens.data_ptr(), None if mask is None else mask.data_ptr(),
                B, L, ws.data_ptr(), out.data_ptr())
        with torch.cuda.device(ids.device):
            if dropout is None:
                _lib.check(self.lib.ance_encoder_forward_train(*args, _lib.current_stream()))
            else:
                p_hidden, p_attn, seed = dropout
                _lib.check(self.lib.ance_encoder_forward_train_dropout(*args, float(p_hidden), float(p_attn), int(seed),
                                                                       _lib.current_stream()))
        return out, ws

    def forward_train_packed(self, ids: torch.Tensor, lens: torch.Tensor, lens_host: torch.Tensor,
                             dropout: Optional[tuple] = None, align: int = 16):
        """forward_train() of a [B, L] batch whose row b is the non-empty prefix of lens[b] tokens, computing the real
        tokens only (ance_encoder_forward_train_packed): lens int32 [B] on the device and lens_host the same on the host;
        align 16 gives forward_train's output bit for bit, 1 packs densest.  -> (out fp32 [B, H], workspace tensor)."""
        B, L = ids.shape
        lens_host = lens_host.to(torch.int32).contiguous()
        self.set_param("varlen_align", align)
        n = C.c_size_t()
        _lib.check(self.lib.ance_encoder_train_workspace_packed(self.h, lens_host.data_ptr(), B, L, C.byref(n)))
        ws = torch.empty(n.value, dtype=torch.uint8, device=ids.device)
        out = torch.empty((B, self.hidden_size), dtype=torch.float32, device=ids.device)
        p_hidden, p_attn, seed = dropout if dropout is not None else (0.0, 0.0, 0)
        with torch.cuda.device(ids.device):
            _lib.check(self.lib.ance_encoder_forward_train_packed(
                self.h, ids.data_ptr(), lens.data_ptr(), lens_host.data_ptr(), B, L, ws.data_ptr(), out.data_ptr(),
                float(p_hidden), float(p_attn), int(seed), _lib.current_stream()))
        return out, ws

    def backward(self, d_out: torch.Tensor, ws: torch.Tensor, grads) -> None:
        """Gradients of sum(d_out * out) for the forward_train that filled `ws`, written into `grads` (fp32 tensors
        grouped as _param_groups)."""
        w, lw = _fill(_lib.EncoderGrads, _lib.LayerGrads, grads, _dev_ptr)
        with torch.cuda.device(d_out.device):
            _lib.check(self.lib.ance_encoder_backward(self.h, d_out.data_ptr(), ws.data_ptr(), C.byref(w),
                                                      _lib.current_stream()))


class _TrainableEncode(torch.autograd.Function):
    """Embeddings [B, H] of a batch as a function of the encoder's parameters (the `params` inputs, in _param_groups
    order), so that their .grad accumulates and DDP's hooks fire.  packed = (lens_host, align): the packed forward of
    prefix rows of lens (forward_train_packed); None: the dense forward."""

    @staticmethod
    def forward(ctx, enc, n_layer, ids, lens, mask, dropout, packed, *params):
        if packed is None:
            out, ws = enc.forward_train(ids, lens, mask, dropout)
        else:
            out, ws = enc.forward_train_packed(ids, lens, packed[0], dropout, packed[1])
        ctx.enc, ctx.ws, ctx.n_layer = enc, ws, n_layer
        ctx.shapes = [p.shape for p in params]
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_out):
        dev = ctx.ws.device
        flat = [torch.empty(s, dtype=torch.float32, device=dev) for s in ctx.shapes]
        n = ctx.n_layer
        groups = (flat[:5], [flat[5 + 16 * i:5 + 16 * (i + 1)] for i in range(n)], flat[5 + 16 * n:])
        ctx.enc.backward(d_out.float().contiguous(), ctx.ws, groups)
        return (None, None, None, None, None, None, None, *flat)


def _forward_varlen(self, ids: torch.Tensor, lens: torch.Tensor, lens_host: Optional[torch.Tensor] = None,
                    out: Optional[torch.Tensor] = None, align: int = 1) -> torch.Tensor:
    """ids int32 [B, L <= 128] CUDA, lens int32 [B] CUDA (+ the same lengths on the host, else they are copied back):
    only the real tokens are computed (ance_encoder_forward_varlen).  -> fp32 [B, H]."""
    return _forward_plan(self, self.lib.ance_encoder_forward_varlen, ids, lens, lens_host, out, align)


def _forward_packed(self, ids: torch.Tensor, lens: torch.Tensor, lens_host: Optional[torch.Tensor] = None,
                    out: Optional[torch.Tensor] = None, align: int = 1) -> torch.Tensor:
    """ids int32 [B, L <= 512] CUDA, lens int32 [B] CUDA, each in [1, L] (+ the same lengths on the host, else they are
    copied back): only the real tokens are computed, sequences of up to 512 tokens (ance_encoder_forward_packed).
    align = 16: bit-identical to forward() at the same L; align = 1: densest packing.  -> fp32 [B, H]."""
    return _forward_plan(self, self.lib.ance_encoder_forward_packed, ids, lens, lens_host, out, align)


def _forward_plan(self, entry, ids, lens, lens_host, out, align):
    B, L = ids.shape
    if out is None:
        out = torch.empty((B, self.hidden_size), dtype=torch.float32, device=ids.device)
    elif out.shape != (B, self.hidden_size) or out.dtype != torch.float32 or not out.is_contiguous() or out.device != ids.device:
        raise ValueError("out must be a contiguous float32 tensor [B, hidden] on the inputs' device")
    if lens_host is None:
        lens_host = lens.cpu()
    lens_host = lens_host.to(torch.int32).contiguous()
    if lens_host.device.type != "cpu" or lens_host.shape != (B,):
        raise ValueError("lens_host must be a CPU tensor [B]")
    self.set_param("varlen_align", align)
    with torch.cuda.device(ids.device):
        _lib.check(entry(self.h, ids.data_ptr(), lens.data_ptr(), lens_host.data_ptr(), B, L, out.data_ptr(),
                         _lib.current_stream()))
    return out


_CudaEncoder.forward_varlen = _forward_varlen
_CudaEncoder.forward_packed = _forward_packed


class _B200Encoder(nn.Module):
    """Common machinery: lazily (re)build the CUDA encoder when the parameters move or change."""

    #: tokens processed per launch sequence (activations: ~14 KB per token).  75,776 = 592 row blocks of 128 (the GEMM's
    #: row tile); about 1 GB of activations.
    max_tokens = int(os.environ.get("ANCE_B200_MAX_TOKENS", 75776))

    #: 16-bit storage format of weights and activations inside the CUDA encoder: "fp16" (11 significant bits; the
    #: embeddings land within ~1e-2 of the reference's fp32 forward) or "bf16" (8 bits, for a checkpoint whose
    #: activations leave the fp16 range — `check_inputs()` raises on the non-finite embeddings that produces).
    #: Same tensor-core rate either way.
    encoder_operand = os.environ.get("ANCE_B200_ENCODER_OPERAND", "fp16")

    #: set_trainable(True): embeddings computed while grad is enabled carry an autograd graph (dense, L <= _train_max_len)
    _trainable = False
    _train_max_len = 128
    _dropout = (0.0, 0.0)   # (hidden, attention-probability) rates of the trainable forward in train() mode
    _packed = False         # set_trainable(..., packed=True): prefix-mask batches train through the packed forward

    def _default_dropout(self) -> tuple:
        """dropout=True: the checkpoint config's hidden_dropout_prob / attention_probs_dropout_prob."""
        return (float(self.config.hidden_dropout_prob), float(self.config.attention_probs_dropout_prob))

    def set_trainable(self, on: bool = True, max_len: int = 128, dropout=False, packed: bool = False):
        """Opt in to gradients: while torch grad mode is on, query_emb / body_emb / encode_lens (dense batches of up to
        `max_len` tokens per sequence or MaxP chunk: 8, 16, 32, 64 or 128, or a multiple of 128 up to max_len) and the
        triplet forward() return tensors whose backward runs the encoder's backward kernels; the other encode paths raise
        instead of returning detached results.  max_len is 128, 256, 384 or 512.  Off by default.

        dropout: False (default) trains the eval-mode forward; True applies the reference's training-mode dropout with the
        rates of the config (RoBERTa: hidden_dropout_prob / attention_probs_dropout_prob; the DPR BiEncoder: 0.1 / 0.1);
        a float sets both rates.  Dropout is applied only on the gradient path and only while the module is in train()
        mode (from_pretrained ends in eval()); each encode draws its mask seed from torch's default CPU generator, so
        torch.manual_seed reproduces a step.

        packed: False (default) trains the padded [B, L] batch.  True computes the real tokens only: an encode whose rows
        each have a non-empty prefix mask (as the token caches produce) runs as ONE packed training forward and backward
        (varlen_align 16: the same embeddings, dropout masks and loss as the dense path; gradients equal up to fp32
        summation order), with its lengths from one device-to-host copy.  Other encodes are split: the prefix rows go
        packed, rows of no real token whose ids are all padding share one dense encode of such a row (MaxP's empty
        chunks), any other row takes the dense path.  Such a split encode gives the dense path's values without dropout;
        with dropout each part draws its own seed and numbers its sequences from 0, and the empty chunks share one mask,
        so its masks are not the padded batch's.  L may be any length up to max_len, and encode_lens_packed becomes
        trainable.  A batch must fit one plan of max_tokens rows."""
        if max_len not in (128, 256, 384, 512):
            raise ValueError(f"max_len must be 128, 256, 384 or 512, got {max_len!r}")
        if dropout is True:
            rates = self._default_dropout()
        elif dropout is False or dropout is None:
            rates = (0.0, 0.0)
        else:
            rates = (float(dropout), float(dropout))
        if not all(0.0 <= r < 1.0 for r in rates):
            raise ValueError(f"dropout rates must be in [0, 1), got {rates!r}")
        self._trainable = bool(on)
        self._train_max_len = int(max_len)
        self._dropout = rates
        self._packed = bool(packed)
        return self

    def _train_dropout(self) -> Optional[tuple]:
        """(p_hidden, p_attn, seed) for one trainable encode, or None (no dropout configured, or eval() mode)."""
        if not self.training or self._dropout == (0.0, 0.0):
            return None
        lo, hi = torch.randint(0, 2 ** 32, (2,), dtype=torch.int64).tolist()
        return self._dropout + (lo | (hi << 32),)

    def _grad_path(self) -> bool:
        return self._trainable and torch.is_grad_enabled()

    def _refuse_grad(self, what: str) -> None:
        if self._grad_path():
            raise _lib.AnceError(f"{what} has no backward: trainable encoders take dense batches of up to max_len = "
                                 f"{self._train_max_len} tokens through query_emb / body_emb / encode_lens (or run this "
                                 "under torch.no_grad())")

    def _train_emb(self, enc, backbone, head, ids, lens, mask, align: int = 16):
        B, L = ids.shape
        max_len = self._train_max_len
        if L > max_len:
            raise _lib.AnceError(f"inputs of {L} tokens have no backward: the trainable encoder covers up to max_len = "
                                 f"{max_len} tokens (set_trainable(True, max_len=...) takes 128, 256, 384 or 512; or run "
                                 "longer inputs under torch.no_grad())")
        if self._packed:
            return self._train_emb_routed(enc, backbone, head, ids, lens, mask, align)
        return self._train_emb_dense(enc, backbone, head, ids, lens, mask)

    def _train_params(self, enc, backbone, head):
        """Refresh the handle from the parameters; -> (number of layers, the parameters in _param_groups order)."""
        # The device weights are refreshed from the parameters before every training forward, whatever their `_version`
        # says: optimizers that write through `p.data` (the reference trainer's Lamb, transformers' AdamW) do not bump it.
        if not enc.update_weights(backbone, head):
            raise _lib.AnceError("a trainable encoder needs contiguous fp32 parameters on the inputs' device")
        max_len = self._train_max_len
        if getattr(enc, "_train_max_len", 128) != max_len:
            enc.set_param("train_max_len", max_len)
            enc._train_max_len = max_len
        embs, layers, hd = _param_groups(backbone, head)
        return len(layers), embs + [t for l in layers for t in l] + hd

    def _train_emb_routed(self, enc, backbone, head, ids, lens, mask, align):
        """packed=True: prefix rows through the packed forward, all-padding rows through one dense encode of such a row,
        the rest through the dense path; one device-to-host copy of the lengths (and prefix flags)."""
        B, L = ids.shape
        dev = ids.device
        if lens is None:
            m = mask != 0
            lens_d = m.sum(dim=1, dtype=torch.int32)
            prefix = (m == (torch.arange(L, device=dev)[None, :] < lens_d[:, None])).all(dim=1)
            lh, pre = torch.stack([lens_d, prefix.to(torch.int32)]).cpu()
        else:
            lh = lens.cpu()
            pre = torch.ones(B, dtype=torch.int32)
        ok = (pre != 0) & (lh >= 1) & (lh <= L)
        tp = n_layer, params = self._train_params(enc, backbone, head)   # one weight refresh for all the sub-encodes
        if bool(ok.all()):
            lh32 = lh.to(torch.int32)
            return _TrainableEncode.apply(enc, n_layer, ids, lh32.to(dev), None, self._train_dropout(), (lh32, align),
                                          *params)
        parts = []
        sel = torch.nonzero(ok).flatten()
        if sel.numel():
            lh32 = lh[sel].to(torch.int32)
            sd = sel.to(dev)
            parts.append((sel, _TrainableEncode.apply(enc, n_layer, ids[sd].contiguous(), lh32.to(dev), None,
                                                      self._train_dropout(), (lh32, align), *params)))
        rest = torch.nonzero(~ok).flatten()
        rd = rest.to(dev)
        allpad = (lh[rest] == 0) & (ids[rd] == enc.pad_id).all(dim=1).cpu()
        pad_rows, other = rest[allpad], rest[~allpad]
        if pad_rows.numel():   # every all-padding row has the same embedding: one encode, broadcast
            one = ids[rd[allpad.to(dev)][:1]].contiguous()
            z = None if lens is None else torch.zeros(1, dtype=lens.dtype, device=dev)
            zm = None if mask is None else torch.zeros((1, L), dtype=mask.dtype, device=dev)
            emb = self._train_emb_dense(enc, backbone, head, one, z, zm, tp)
            parts.append((pad_rows, emb.expand(pad_rows.numel(), emb.shape[1])))
        if other.numel():
            od = other.to(dev)
            parts.append((other, self._train_emb_dense(enc, backbone, head, ids[od].contiguous(),
                                                       None if lens is None else lens[od].contiguous(),
                                                       None if mask is None else mask[od].contiguous(), tp)))
        order = torch.cat([p[0] for p in parts])
        inv = torch.empty_like(order)
        inv[order] = torch.arange(B)
        return torch.cat([p[1] for p in parts])[inv.to(dev)]

    def _train_emb_dense(self, enc, backbone, head, ids, lens, mask, tp=None):
        """tp: (n_layer, params) of a _train_params call already made for this encode (else it is made here)."""
        B, L = ids.shape
        if L > 128 and L % 128:
            raise _lib.AnceError(f"inputs of {L} tokens have no backward: above 128 tokens the trainable encoder takes "
                                 "multiples of 128 (pad the batch to 256, 384 or 512)")
        if B * L > enc.max_tokens:
            raise _lib.AnceError(f"a trainable batch of {B} x {L} tokens exceeds max_tokens {enc.max_tokens}")
        n_layer, params = tp if tp is not None else self._train_params(enc, backbone, head)
        return _TrainableEncode.apply(enc, n_layer, ids, lens, mask, self._train_dropout(), None, *params)

    def _enc_for(self, name, backbone, arch, heads, pad_id, head, device) -> _CudaEncoder:
        if device.type != "cuda":
            raise _lib.AnceError("ance_b200 models run on an sm_90 GPU only (no CPU fallback): move the model and "
                                 "the inputs to a CUDA device")
        cache = self.__dict__.setdefault("_enc_cache", {})
        # Rebuild the device copy when a parameter was written in place (load_state_dict / optimizer step bump
        # `_version`) or the module moved (`.to()` swaps `.data`: new storage).  The Parameter objects themselves are
        # stable, so the module tree is walked once and ~200 version counters are summed per call, not re-collected.
        params = cache.get("_params")
        if params is None:
            params = cache["_params"] = list(self.parameters())
        ver = (sum(p._version for p in params), params[0].data_ptr(), str(device), self.encoder_operand)
        hit = cache.get(name)
        if hit is not None and hit[0] != ver and hit[0][1:] == ver[1:] and hit[1].update_weights(backbone, head):
            cache[name] = (ver, hit[1])   # only values changed (optimizer step, load_state_dict): refreshed in place
        elif hit is None or hit[0] != ver:
            cache[name] = (ver, _CudaEncoder(backbone, arch, heads, pad_id, head, self.max_tokens, device,
                                             self.encoder_operand))
        return cache[name][1]

    def _emb_packed(self, name, backbone, arch, heads, pad_id, head, input_ids, align, ids_host):
        """Same result as the dense forward with the mask input_ids != pad_id at the cost of the real tokens: rows whose
        non-padding ids form a non-empty prefix go through the packed forward, the others through the dense one with
        that mask.  The lengths are read from `ids_host` (the host copy of input_ids; copied back when not given)."""
        self._refuse_grad("query_emb_packed / body_emb_packed")
        if input_ids.device.type != "cuda":
            raise _lib.AnceError("ance_b200 models run on an sm_90 GPU only (no CPU fallback)")
        ids = input_ids.to(torch.int32).contiguous()
        B, L = ids.shape
        nz = (ids_host if ids_host is not None else input_ids.cpu()).reshape(B, L) != pad_id
        lens = nz.sum(dim=1)
        ok = (nz == (torch.arange(L)[None, :] < lens[:, None])).all(dim=1) & (lens > 0)
        enc = self._enc_for(name, backbone, arch, heads, pad_id, head, ids.device)
        lens32 = lens.to(torch.int32)
        if bool(ok.all()):
            return enc.forward_packed(ids, lens32.to(ids.device), lens32, align=align)
        out = torch.empty((B, enc.hidden_size), dtype=torch.float32, device=ids.device)
        sel, rest = torch.nonzero(ok).flatten(), torch.nonzero(~ok).flatten()
        if sel.numel():
            sd = sel.to(ids.device)
            out[sd] = enc.forward_packed(ids[sd].contiguous(), lens32[sel].to(ids.device), lens32[sel].contiguous(),
                                         align=align)
        rd = rest.to(ids.device)
        out[rd] = enc.forward(ids[rd].contiguous(), None, (ids[rd] != pad_id).to(torch.uint8).contiguous())
        return out

    def check_inputs(self) -> None:
        """Deferred input validation (keeps `body_emb`/`query_emb` asynchronous): raises if any encode since the last
        call saw a token id outside the vocabulary or a position beyond max_position_embeddings, where the reference's
        nn.Embedding lookup raises an IndexError.  Synchronises the current stream; the drivers call it per pass."""
        for key, val in self.__dict__.get("_enc_cache", {}).items():
            if key != "_params":
                val[1].check()

    @staticmethod
    def _prep(input_ids, attention_mask):
        if input_ids.device.type != "cuda":
            raise _lib.AnceError("ance_b200 models run on an sm_90 GPU only (no CPU fallback)")
        ids = input_ids.to(torch.int32).contiguous()
        mask = (attention_mask != 0).to(torch.uint8).contiguous()
        return ids, mask

    # -- reference `NLL.forward` (model/models.py:58-84) ------------------------------------------------------
    # Same signature and return values as the reference: embeddings when only one side is given, `(loss,)` for a
    # (query, positive, negative) triplet batch.  After set_trainable(True), with grad enabled, the loss carries an
    # autograd graph through the encoder's backward kernels (inputs of up to max_len tokens); otherwise it is computed
    # under no_grad, as the value the trainer logs.
    @staticmethod
    def _pair_logits(q_embs, x_embs, input_ids_x, attention_mask_x):
        return (q_embs * x_embs).sum(-1)

    def forward(self, query_ids, attention_mask_q, input_ids_a=None, attention_mask_a=None, input_ids_b=None,
                attention_mask_b=None, is_query=True):
        with contextlib.nullcontext() if self._grad_path() else torch.no_grad():
            return self._nll_forward(query_ids, attention_mask_q, input_ids_a, attention_mask_a, input_ids_b,
                                     attention_mask_b, is_query)

    def _nll_forward(self, query_ids, attention_mask_q, input_ids_a, attention_mask_a, input_ids_b, attention_mask_b,
                     is_query):
        if input_ids_b is None and is_query:
            return self.query_emb(query_ids, attention_mask_q)
        if input_ids_b is None:
            return self.body_emb(query_ids, attention_mask_q)
        q_embs = self.query_emb(query_ids, attention_mask_q)
        a_embs = self.body_emb(input_ids_a, attention_mask_a)
        b_embs = self.body_emb(input_ids_b, attention_mask_b)
        logit_matrix = torch.stack([self._pair_logits(q_embs, a_embs, input_ids_a, attention_mask_a),
                                    self._pair_logits(q_embs, b_embs, input_ids_b, attention_mask_b)], dim=1)  # [B, 2]
        loss = -torch.log_softmax(logit_matrix, dim=1)[:, 0]
        return (loss.mean(),)


# ---------------------------------------------------------------------------------------------
# rdot_nll / rdot_nll_multi_chunk
# ---------------------------------------------------------------------------------------------
class RobertaDot_NLL_LN(_B200Encoder):
    """model/models.py:137-157: RoBERTa -> CLS -> Linear(hidden, 768) -> LayerNorm(768)."""

    def __init__(self, config, model_argobj=None):
        super().__init__()
        self.config = config
        self.use_mean = False if model_argobj is None else model_argobj.use_mean  # models.py:24-28
        if self.use_mean:
            raise NotImplementedError("use_mean=True is never registered by the reference (models.py:302-316)")
        self.roberta = _backbone(config.vocab_size, config.hidden_size, config.num_hidden_layers,
                                 config.intermediate_size, config.max_position_embeddings, config.type_vocab_size,
                                 config.pad_token_id, config.layer_norm_eps)
        self.embeddingHead = nn.Linear(config.hidden_size, 768)
        self.norm = nn.LayerNorm(768)
        self.apply(self._init_weights)

    @staticmethod
    def _init_weights(module):
        if isinstance(module, (nn.Linear, nn.Embedding)):  # models.py:31-36
            module.weight.data.normal_(mean=0.0, std=0.02)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, *model_args, config=None, from_tf=False, cache_dir=None,
                        **kwargs):
        if from_tf:
            raise NotImplementedError("TensorFlow checkpoints are not supported")
        path = str(pretrained_model_name_or_path)
        if config is None:
            from transformers import RobertaConfig
            config = RobertaConfig.from_pretrained(path)
        return _load_checkpoint(cls(config), path)  # classifier.*, pooler.*: unused (SURVEY §8 a2)

    def _encoder(self, device):
        return self._enc_for("roberta", self.roberta, _lib.ANCE_ARCH_ROBERTA, self.config.num_attention_heads,
                             self.config.pad_token_id, (self.embeddingHead, self.norm), device)

    def query_emb(self, input_ids, attention_mask):
        ids, mask = self._prep(input_ids, attention_mask)
        if self._grad_path():
            return self._train_emb(self._encoder(ids.device), self.roberta, (self.embeddingHead, self.norm), ids, None,
                                   mask)
        return self._encoder(ids.device).forward(ids, None, mask)

    def body_emb(self, input_ids, attention_mask):
        return self.query_emb(input_ids, attention_mask)

    # fast path used by the GPU refresher: mask given as lengths (msmarco_data.py:282 form)
    def encode_lens(self, ids_i32: torch.Tensor, lens_i32: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        if self._grad_path() and out is None:
            return self._train_emb(self._encoder(ids_i32.device), self.roberta, (self.embeddingHead, self.norm),
                                   ids_i32.contiguous(), lens_i32.contiguous(), None)
        self._refuse_grad("encode_lens(out=...)")
        return self._encoder(ids_i32.device).forward(ids_i32.contiguous(), lens_i32.contiguous(), None, out=out)

    def encode_lens_varlen(self, ids_i32: torch.Tensor, lens_i32: torch.Tensor, lens_host: Optional[torch.Tensor] = None,
                           out: Optional[torch.Tensor] = None, align: int = 1) -> torch.Tensor:
        """encode_lens at the cost of the REAL tokens only: whole sequences of any length are packed into 128-token
        attention tiles.  align = 1: densest packing, embeddings equal encode_lens up to fp32 summation order inside a
        tile; align = 16: bit-identical to encode_lens and independent of the batch composition (~12 % fewer real tokens
        per tile).  L <= 128 (the MS MARCO passage and query caches); longer caches use encode_lens_bucketed."""
        self._refuse_grad("encode_lens_varlen")
        return self._encoder(ids_i32.device).forward_varlen(ids_i32.contiguous(), lens_i32.contiguous(), lens_host, out=out,
                                                            align=align)

    def encode_lens_packed(self, ids_i32: torch.Tensor, lens_i32: torch.Tensor, lens_host: Optional[torch.Tensor] = None,
                           out: Optional[torch.Tensor] = None, align: Optional[int] = None) -> torch.Tensor:
        """encode_lens at the cost of the REAL tokens only, for any L <= 512 (lengths in [1, L]).  align = 16: bit-identical
        to encode_lens at the same L, whatever else is in the batch; align = 1: densest packing, equal up to fp32
        summation order.  align None: 1 for inference, 16 on the trainable path (set_trainable(..., packed=True) with
        grad enabled), where attention dropout needs it.  L <= 128 is encode_lens_varlen."""
        if self._grad_path() and self._packed and out is None:
            if lens_host is not None:
                raise _lib.AnceError("the trainable encode_lens_packed reads the lengths itself: pass lens_host=None")
            return self._train_emb(self._encoder(ids_i32.device), self.roberta, (self.embeddingHead, self.norm),
                                   ids_i32.contiguous(), lens_i32.contiguous(), None, 16 if align is None else align)
        self._refuse_grad("encode_lens_packed")
        return self._encoder(ids_i32.device).forward_packed(ids_i32.contiguous(), lens_i32.contiguous(), lens_host, out=out,
                                                            align=1 if align is None else align)

    def encode_lens_bucketed(self, ids_i32: torch.Tensor, lens_i32: torch.Tensor, min_bucket: int = 16,
                             out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Same result as encode_lens, without the FLOPs of all-padding tails: sequences are grouped by the
        smallest supported padded length >= their own length (16/32/64/128/256/384/512) and each group is
        encoded at that length.  Padding keys carry the additive -10000 (probability exactly 0 in fp32) and
        padding rows are never read, so dropping trailing pad columns does not change a sequence's embedding."""
        self._refuse_grad("encode_lens_bucketed")
        B, L = ids_i32.shape
        buckets = [b for b in (8, 16, 32, 64) if min_bucket <= b < L] + [b for b in range(128, L + 1, 128)]
        if not buckets or buckets[-1] != L:
            buckets.append(L)
        bt = torch.tensor(buckets, device=lens_i32.device, dtype=torch.int32)
        which = torch.bucketize(lens_i32.clamp(min=1), bt)  # first bucket with capacity >= len
        if out is None:
            out = torch.empty((B, 768), dtype=torch.float32, device=ids_i32.device)
        for bi, Lb in enumerate(buckets):
            sel = torch.nonzero(which == bi).flatten()
            if sel.numel() == 0:
                continue
            out[sel] = self.encode_lens(ids_i32[sel, :Lb].contiguous(), lens_i32[sel].contiguous())
        return out


class RobertaDot_CLF_ANN_NLL_MultiChunk(RobertaDot_NLL_LN):
    """model/models.py:160-199: documents are 4 independent 512-token chunks; one vector per chunk."""

    def __init__(self, config):
        super().__init__(config)
        self.base_len = 512

    def body_emb(self, input_ids, attention_mask):
        """[B, chunks * 512] -> [B, chunks, 768]; trainable (every chunk through the dense backward) with max_len >= 512."""
        if self._train_max_len < self.base_len:
            self._refuse_grad("the multi-chunk body_emb (its 512-token chunks need set_trainable(True, max_len=512))")
        batchS, full_length = input_ids.shape
        chunk_factor = full_length // self.base_len
        if chunk_factor == 0 or full_length % chunk_factor != 0:
            raise ValueError(f"document length {full_length} is not a multiple of base_len {self.base_len}")
        seq = full_length // chunk_factor
        ids, mask = self._prep(input_ids.reshape(batchS * chunk_factor, seq),
                               attention_mask.reshape(batchS * chunk_factor, seq))
        if self._grad_path():
            emb = self._train_emb(self._encoder(ids.device), self.roberta, (self.embeddingHead, self.norm), ids, None, mask)
        else:
            emb = self._encoder(ids.device).forward(ids, None, mask)
        return emb.reshape(batchS, chunk_factor, emb.shape[-1])

    def _pair_logits(self, q_embs, x_embs, input_ids_x, attention_mask_x):
        """MaxP (models.py:87-134): best chunk of the document; a chunk whose FIRST token is padding gets -9999."""
        batchS, full_length = input_ids_x.shape
        chunk_factor = full_length // self.base_len
        first = attention_mask_x.reshape(batchS, chunk_factor, -1)[:, :, 0]
        inverted_bias = ((1 - first) * (-9999)).float()
        scores = torch.matmul(q_embs.unsqueeze(1), x_embs.transpose(1, 2))[:, 0, :]   # [B, chunks]
        return (scores + inverted_bias).max(dim=-1).values

    def encode_lens_multi_chunk(self, ids_i32: torch.Tensor, lens_i32: torch.Tensor) -> torch.Tensor:
        """[B, full] ids + document lengths -> [B, chunks, 768]; chunk c sees max(0, min(512, len - 512c)) tokens."""
        self._refuse_grad("encode_lens_multi_chunk")
        B, full = ids_i32.shape
        cf = full // self.base_len
        seq = full // cf
        off = torch.arange(cf, device=ids_i32.device, dtype=torch.int32) * seq
        clen = (lens_i32[:, None] - off[None, :]).clamp_(0, seq).to(torch.int32).reshape(-1)
        emb = self._encoder(ids_i32.device).forward(ids_i32.reshape(B * cf, seq).contiguous(), clen.contiguous(), None)
        return emb.reshape(B, cf, emb.shape[-1])

    def encode_lens_multi_chunk_packed(self, ids_i32: torch.Tensor, lens_i32: torch.Tensor,
                                       lens_host: Optional[torch.Tensor] = None, align: int = 1) -> torch.Tensor:
        """encode_lens_multi_chunk (same [B, chunks, 768]) at the cost of the real tokens: the chunks with tokens go through
        the packed forward (align as in encode_lens_packed; 16 = bit-identical); an all-padding chunk (length 0, every id
        pad_id, as the token caches store them) gets the one vector such a chunk has, computed once per encoder and
        weights by the dense forward; any other empty chunk is encoded densely."""
        self._refuse_grad("encode_lens_multi_chunk_packed")
        B, full = ids_i32.shape
        cf = full // self.base_len
        seq = full // cf
        dev = ids_i32.device
        if lens_host is None:
            lens_host = lens_i32.cpu()
        lh = lens_host.to(torch.int64).reshape(B)
        clen = (lh[:, None] - torch.arange(cf, dtype=torch.int64)[None, :] * seq).clamp_(0, seq).reshape(-1)
        ids2 = ids_i32.reshape(B * cf, seq).contiguous()
        enc = self._encoder(dev)
        out = torch.empty((B * cf, 768), dtype=torch.float32, device=dev)
        real = torch.nonzero(clen > 0).flatten()
        if real.numel() == B * cf:
            return enc.forward_packed(ids2, clen.to(torch.int32).to(dev), clen.to(torch.int32), out=out,
                                      align=align).reshape(B, cf, 768)
        if real.numel():
            rl = clen[real].to(torch.int32)
            rd = real.to(dev)
            out[rd] = enc.forward_packed(ids2[rd].contiguous(), rl.to(dev), rl, align=align)
        empty = torch.nonzero(clen == 0).flatten().to(dev)
        allpad = (ids2[empty] == self.config.pad_token_id).all(dim=1).cpu()
        pad_rows, other = empty[allpad.to(dev)], empty[~allpad.to(dev)]
        if pad_rows.numel():
            out[pad_rows] = self._allpad_row(enc, seq)
        if other.numel():
            out[other] = enc.forward(ids2[other].contiguous(), torch.zeros(other.numel(), dtype=torch.int32, device=dev),
                                     None)
        return out.reshape(B, cf, 768)

    def _allpad_row(self, enc, seq: int) -> torch.Tensor:
        """The embedding of an all-padding chunk of `seq` tokens (dense forward), cached on the encoder handle, which is
        rebuilt whenever the weights change."""
        cache = enc.__dict__.setdefault("_allpad", {})
        if seq not in cache:
            ids = torch.full((1, seq), self.config.pad_token_id, dtype=torch.int32, device=enc.device)
            cache[seq] = enc.forward(ids, torch.zeros(1, dtype=torch.int32, device=enc.device), None)[0]
        return cache[seq]


# ---------------------------------------------------------------------------------------------
# dpr
# ---------------------------------------------------------------------------------------------
class _BertDims:
    vocab_size, hidden_size, num_hidden_layers, intermediate_size = 30522, 768, 12, 3072
    max_position_embeddings, type_vocab_size, pad_token_id, layer_norm_eps, num_attention_heads = 512, 2, 0, 1e-12, 12


class BiEncoder(_B200Encoder):
    """model/models.py:243-259: separate question / ctx BERT-base encoders, CLS of the last layer, no head.
    The reference initialises both from "bert-base-uncased" (models.py:228-233) and then overwrites every
    tensor from the DPR checkpoint (run_ann_data_gen_dpr.py:119-124); there is no network here, so the
    skeleton is created with bert-base-uncased's dimensions and the checkpoint provides the values."""

    def __init__(self, args=None):
        super().__init__()

        class d(_BertDims):  # bert-base-uncased unless `args` overrides a dimension (tests use small models)
            num_hidden_layers = getattr(args, "num_hidden_layers", _BertDims.num_hidden_layers)
            vocab_size = getattr(args, "vocab_size", _BertDims.vocab_size)

        self.dims = d
        self.question_model = _backbone(d.vocab_size, d.hidden_size, d.num_hidden_layers, d.intermediate_size,
                                        d.max_position_embeddings, d.type_vocab_size, d.pad_token_id, d.layer_norm_eps)
        self.ctx_model = _backbone(d.vocab_size, d.hidden_size, d.num_hidden_layers, d.intermediate_size,
                                   d.max_position_embeddings, d.type_vocab_size, d.pad_token_id, d.layer_norm_eps)

    def set_trainable(self, on: bool = True, max_len: Optional[int] = None, dropout=False, packed: bool = False):
        """As _B200Encoder.set_trainable for both BERT encoders; training needs an explicit max_len (DPR's inputs are 256
        tokens: set_trainable(True, max_len=256)).  dropout=True is HFBertEncoder.init_encoder's default rate, 0.1.
        packed=True: prefix-mask rows (mask input_ids != 0) train through the packed forward."""
        if on and max_len is None:
            raise NotImplementedError("the DPR BiEncoder trains on 256-token inputs: call set_trainable(True, max_len=256) "
                                      "(or 128 / 384 / 512 for other input lengths)")
        return super().set_trainable(on, 128 if max_len is None else max_len, dropout, packed)

    def _default_dropout(self) -> tuple:
        return (0.1, 0.1)   # model/models.py:229-233, init_encoder(dropout=0.1)

    def load_state_dict(self, state_dict, strict=True, **kw):
        # HF BertModel checkpoints carry pooler.* and position_ids buffers the path never uses
        own = self.state_dict()
        sd = {k: v for k, v in state_dict.items() if k in own}
        missing = [k for k in own if k not in sd]
        if missing and strict:
            raise KeyError(f"DPR checkpoint lacks {len(missing)} tensors, e.g. {missing[:3]}")
        return super().load_state_dict(sd, strict=False)

    def _emb(self, name, backbone, input_ids, attention_mask):
        ids, mask = self._prep(input_ids, attention_mask)
        enc = self._enc_for(name, backbone, _lib.ANCE_ARCH_BERT, self.dims.num_attention_heads, 0, None, ids.device)
        if self._grad_path():
            return self._train_emb(enc, backbone, None, ids, None, mask)
        return enc.forward(ids, None, mask)

    def query_emb(self, input_ids, attention_mask):
        return self._emb("question", self.question_model, input_ids, attention_mask)

    def body_emb(self, input_ids, attention_mask):
        return self._emb("ctx", self.ctx_model, input_ids, attention_mask)

    #: the refresher encodes DPR caches with the mask input_ids != 0 (DPR_data.py:283)
    mask_pad_id = 0

    def query_emb_packed(self, input_ids, align: int = 1, ids_host: Optional[torch.Tensor] = None):
        """query_emb(input_ids, input_ids != 0) computing the real tokens only (align: see encode_lens_packed)."""
        return self._emb_packed("question", self.question_model, _lib.ANCE_ARCH_BERT, self.dims.num_attention_heads, 0,
                                None, input_ids, align, ids_host)

    def body_emb_packed(self, input_ids, align: int = 1, ids_host: Optional[torch.Tensor] = None):
        """body_emb(input_ids, input_ids != 0) computing the real tokens only (align: see encode_lens_packed)."""
        return self._emb_packed("ctx", self.ctx_model, _lib.ANCE_ARCH_BERT, self.dims.num_attention_heads, 0, None,
                                input_ids, align, ids_host)

    def forward(self, query_ids, attention_mask_q, input_ids_a=None, attention_mask_a=None, input_ids_b=None,
                attention_mask_b=None):
        """model/models.py:253-266: (q, a) embeddings (the in-batch-negative form), or `(loss,)` for triplets.  Both carry
        an autograd graph after set_trainable(True, max_len=...) with grad enabled; otherwise they are computed under
        no_grad."""
        with contextlib.nullcontext() if self._grad_path() else torch.no_grad():
            return self._bi_forward(query_ids, attention_mask_q, input_ids_a, attention_mask_a, input_ids_b,
                                    attention_mask_b)

    def _bi_forward(self, query_ids, attention_mask_q, input_ids_a, attention_mask_a, input_ids_b, attention_mask_b):
        q_embs = self.query_emb(query_ids, attention_mask_q)
        a_embs = self.body_emb(input_ids_a, attention_mask_a)
        if input_ids_b is None:
            return (q_embs, a_embs)
        b_embs = self.body_emb(input_ids_b, attention_mask_b)
        logit_matrix = torch.stack([(q_embs * a_embs).sum(-1), (q_embs * b_embs).sum(-1)], dim=1)
        return ((-torch.log_softmax(logit_matrix, dim=1)[:, 0]).mean(),)


# ---------------------------------------------------------------------------------------------
# seeddot_nll (SEED-Encoder)
# ---------------------------------------------------------------------------------------------
# configuration_seed_encoder.py:71-112: every field of the SEED-Encoder config and its default.  Only the encoder half is
# computed here; the decoder / pretraining fields are kept so that a config.json round-trips unchanged.
_SEED_DEFAULTS = {
    "pad_token_id": 1, "vocab_size": 32769,
    "encoder_layers": 12, "encoder_embed_dim": 768, "encoder_ffn_embed_dim": 3072, "encoder_attention_heads": 12,
    "dropout": 0.1, "attention_dropout": 0.1, "activation_dropout": 0.0, "encoder_layerdrop": 0.0,
    "max_positions": 512, "activation_fn": "gelu", "quant_noise_pq": 0.0, "quant_noise_pq_block_size": 8,
    "train_ratio": "0.5:0.5", "decoder_atten_window": 2, "pooler_activation_fn": "tanh", "pooler_dropout": 0.0,
    "encoder_layers_to_keep": None, "decoder_layers": 3, "decoder_embed_path": None, "decoder_embed_dim": 768,
    "decoder_ffn_embed_dim": 3072, "decoder_attention_heads": 12, "decoder_normalize_before": True,
    "decoder_learned_pos": True, "adaptive_softmax_cutoff": None, "adaptive_softmax_dropout": 0,
    "share_decoder_input_output_embed": True, "share_all_embeddings": True, "no_token_positional_embeddings": False,
    "adaptive_input": False, "no_cross_attention": False, "cross_self_attention": False, "no_scale_embedding": True,
    "layernorm_embedding": True, "tie_adaptive_weights": True, "decoder_layers_to_keep": None,
    "initializer_range": 0.02,
}


class SEEDEncoderConfig(PretrainedConfig):
    """The SEED-Encoder checkpoint config (`model_type` "seed_encoder"), with the reference's field names and defaults.
    `MSMarcoConfigDict["seeddot_nll"].config_class`: a SEED config.json stores only the values that differ from these
    defaults, so it must be read through this class (RobertaConfig would fill in RoBERTa's)."""
    model_type = "seed_encoder"

    def __init__(self, **kwargs):
        own = {k: kwargs.pop(k, v) for k, v in _SEED_DEFAULTS.items()}
        super().__init__(**kwargs)
        for k, v in own.items():
            setattr(self, k, v)
        self.decoder_output_dim = self.decoder_input_dim = self.decoder_embed_dim
        self.decoder_layerdrop = 0
        self.max_source_positions = self.max_target_positions = self.max_positions


class _SeedSentenceEncoder(nn.Module):
    """Parameter skeleton of the SEED-Encoder's `TransformerSentenceEncoder` (transformer_sentence_encoder.py:695-925)
    under its own names and registration order, with no forward of its own.  It is the post-LN RoBERTa computation the
    encoder kernels run (ANCE_ARCH_ROBERTA): no segment embedding (a zero type row stands in: x + 0 is exact), an
    embedding LayerNorm, separate k / v / q / out projections, erf GELU, every LayerNorm at eps 1e-5."""

    ln_eps = 1e-5   # fairseq LayerNorm default (modules.py:30)

    def __init__(self, vocab, hidden, n_layer, ffn, max_pos, pad_id):
        super().__init__()
        self.embed_tokens = nn.Embedding(vocab, hidden, padding_idx=pad_id)
        self.embed_positions = nn.Embedding(max_pos, hidden, padding_idx=pad_id)
        layers = []
        for _ in range(n_layer):
            l = _Holder()
            att = _Holder()
            att.k_proj, att.v_proj, att.q_proj = _linear(hidden, hidden), _linear(hidden, hidden), _linear(hidden, hidden)
            att.out_proj = _linear(hidden, hidden)
            l.self_attn = att
            l.self_attn_layer_norm = nn.LayerNorm(hidden, eps=self.ln_eps)
            l.fc1 = _linear(hidden, ffn)
            l.fc2 = _linear(ffn, hidden)
            l.final_layer_norm = nn.LayerNorm(hidden, eps=self.ln_eps)
            layers.append(l)
        self.layers = nn.ModuleList(layers)
        self.emb_layer_norm = nn.LayerNorm(hidden, eps=self.ln_eps)
        # the kernels' type embedding: one zero row.  Not persistent, so state_dict() keeps the reference's keys; the
        # gradient the backward writes for it is dropped (a buffer takes no gradient).
        self.register_buffer("type_row", torch.zeros(1, hidden), persistent=False)

    def kernel_params(self):
        """(embeddings, layers) in the order of ance_encoder_weights / ance_layer_weights (see _param_groups)."""
        embs = [self.embed_tokens.weight, self.embed_positions.weight, self.type_row, self.emb_layer_norm.weight,
                self.emb_layer_norm.bias]
        layers = []
        for l in self.layers:
            a = l.self_attn
            layers.append([a.q_proj.weight, a.q_proj.bias, a.k_proj.weight, a.k_proj.bias, a.v_proj.weight, a.v_proj.bias,
                           a.out_proj.weight, a.out_proj.bias, l.self_attn_layer_norm.weight, l.self_attn_layer_norm.bias,
                           l.fc1.weight, l.fc1.bias, l.fc2.weight, l.fc2.bias, l.final_layer_norm.weight,
                           l.final_layer_norm.bias])
        return embs, layers


class SEEDEncoderDot_NLL_LN_B200(_B200Encoder):
    """model/models.py:201-221 (`seeddot_nll`) on the sm_90a encoder: SEED-Encoder -> CLS -> Linear(768, 768) ->
    LayerNorm(768).  Parameter names, shapes and order are the reference's (seed_encoder.encoder.sentence_encoder.*,
    the unused classification_heads.*, embeddingHead.*, norm.*), so pytorch_model.bin and optimizer.pt are
    interchangeable with it.

    As in the reference, the attention mask comes from the ids: keys whose id is config.pad_token_id are masked
    (transformer_sentence_encoder.py:878) and the `attention_mask` argument is ignored.  A cache padded with another id
    therefore attends to its padding, as the reference does.  A row made only of padding, where the reference's softmax
    over -inf yields NaN, gets the kernels' uniform-attention vector instead."""

    def __init__(self, config, model_argobj=None):
        super().__init__()
        self.config = config
        self.use_mean = False if model_argobj is None else model_argobj.use_mean  # models.py:24-28
        if self.use_mean:
            raise NotImplementedError("use_mean=True is never registered by the reference (models.py:302-316)")
        if config.activation_fn != "gelu":
            raise NotImplementedError(f"activation_fn={config.activation_fn!r}: the encoder kernels compute the erf GELU "
                                      "('gelu') only")
        if config.quant_noise_pq > 0:
            # q_noise > 0 also inserts a bias-free Linear after the embeddings, applied in eval mode too
            # (transformer_sentence_encoder.py:779-786)
            raise NotImplementedError(f"quant_noise_pq={config.quant_noise_pq}: the encoder kernels have no "
                                      "quantization-noise embedding projection")
        keep = config.encoder_layers_to_keep
        n_layer = len(keep.split(",")) if keep else config.encoder_layers   # modeling_seed_encoder.py:73-74
        H, pad = config.encoder_embed_dim, config.pad_token_id
        se = _SeedSentenceEncoder(config.vocab_size, H, n_layer, config.encoder_ffn_embed_dim,
                                  config.max_positions + pad + 1, pad)   # learned positions offset by pad (modules.py:289)
        self.seed_encoder = _Holder()
        self.seed_encoder.encoder = _Holder()
        self.seed_encoder.encoder.sentence_encoder = se
        self.classification_heads = _Holder()   # registered for the checkpoint's sake; query_emb never reads it
        self.classification_heads.dense = nn.Linear(H, H)
        self.classification_heads.out_proj = nn.Linear(H, config.num_labels)
        self.embeddingHead = nn.Linear(H, 768)
        self.norm = nn.LayerNorm(768)
        self.apply(RobertaDot_NLL_LN._init_weights)   # EmbeddingMixin._init_weights (models.py:31-36)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, *model_args, config=None, from_tf=False, cache_dir=None,
                        **kwargs):
        """config.json (read as SEEDEncoderConfig unless `config` is given) + pytorch_model.bin / model.safetensors.
        Extra tensors (a pretraining checkpoint's decoder / lm_head) are ignored; a missing one raises KeyError."""
        if from_tf:
            raise NotImplementedError("TensorFlow checkpoints are not supported")
        path = str(pretrained_model_name_or_path)
        if config is None:
            config = SEEDEncoderConfig.from_pretrained(path)
        return _load_checkpoint(cls(config), path)

    #: the refresher encodes seeddot_nll caches with the mask input_ids != pad_token_id (see the class docstring)
    @property
    def mask_pad_id(self) -> int:
        return int(self.config.pad_token_id)

    @property
    def _sentence_encoder(self) -> _SeedSentenceEncoder:
        return self.seed_encoder.encoder.sentence_encoder

    def _default_dropout(self) -> tuple:
        """dropout=True: the config's `dropout` (embeddings, attention and FFN outputs) and `attention_dropout`."""
        return (float(self.config.dropout), float(self.config.attention_dropout))

    def _encoder(self, device):
        return self._enc_for("seed", self._sentence_encoder, _lib.ANCE_ARCH_ROBERTA, self.config.encoder_attention_heads,
                             self.mask_pad_id, (self.embeddingHead, self.norm), device)

    def query_emb(self, input_ids, attention_mask=None):
        """CLS embedding with the mask input_ids != pad_token_id; `attention_mask` is ignored, as in the reference."""
        if self._grad_path() and self.training:
            for field in ("activation_dropout", "encoder_layerdrop"):
                if getattr(self.config, field) > 0:
                    raise NotImplementedError(f"{field}={getattr(self.config, field)}: training-mode SEED-Encoder layers "
                                              "with it have no kernel (set it to 0, or call eval())")
        if input_ids.device.type != "cuda":
            raise _lib.AnceError("ance_b200 models run on an sm_90 GPU only (no CPU fallback)")
        ids = input_ids.to(torch.int32).contiguous()
        mask = (ids != self.mask_pad_id).to(torch.uint8)
        enc = self._encoder(ids.device)
        if self._grad_path():
            return self._train_emb(enc, self._sentence_encoder, (self.embeddingHead, self.norm), ids, None, mask)
        return enc.forward(ids, None, mask)

    def body_emb(self, input_ids, attention_mask=None):
        return self.query_emb(input_ids, attention_mask)

    def query_emb_packed(self, input_ids, align: int = 1, ids_host: Optional[torch.Tensor] = None):
        """query_emb computing the real tokens only (align: see RobertaDot_NLL_LN.encode_lens_packed)."""
        return self._emb_packed("seed", self._sentence_encoder, _lib.ANCE_ARCH_ROBERTA,
                                self.config.encoder_attention_heads, self.mask_pad_id, (self.embeddingHead, self.norm),
                                input_ids, align, ids_host)

    def body_emb_packed(self, input_ids, align: int = 1, ids_host: Optional[torch.Tensor] = None):
        return self.query_emb_packed(input_ids, align, ids_host)


def _reference_seed_class():
    """(the reference's own stock-PyTorch class, None) when the reference repository is importable (its directory on
    sys.path, as its scripts arrange with `sys.path += ['../']`), else (None, the import error)."""
    try:
        from model.models import SEEDEncoderDot_NLL_LN as ref_cls   # /root/reference-style checkout
        return ref_cls, None
    except Exception as e:  # ImportError, or the reference's own third-party imports failing
        return None, e


def _seed_unavailable(e):
    return NotImplementedError(
        "seeddot_nll (SEED-Encoder, model/models.py:201-221): the reference's stock module could not be imported "
        "({}: {}) and no config was given.  Pass a SEEDEncoderConfig (or a checkpoint directory to from_pretrained) to "
        "build the sm_90a model, ance_b200.models.SEEDEncoderDot_NLL_LN_B200.".format(type(e).__name__, e))


class SEEDEncoderDot_NLL_LN:
    """model/models.py:201-221 (`seeddot_nll`), the registry's class.  When the reference repository is importable,
    construction and from_pretrained return the reference's own stock-PyTorch module (no GPU acceleration); otherwise
    they build SEEDEncoderDot_NLL_LN_B200, the same model on the sm_90a encoder, from the config or checkpoint given."""

    def __new__(cls, *a, **k):
        ref, err = _reference_seed_class()
        if ref is not None:
            return ref(*a, **k)
        if not a and k.get("config") is None:
            raise _seed_unavailable(err)
        return SEEDEncoderDot_NLL_LN_B200(*a, **k)

    @classmethod
    def from_pretrained(cls, *a, **k):
        ref, err = _reference_seed_class()
        if ref is not None:
            return ref.from_pretrained(*a, **k)
        if not a and k.get("pretrained_model_name_or_path") is None:
            raise _seed_unavailable(err)
        return SEEDEncoderDot_NLL_LN_B200.from_pretrained(*a, **k)


# ---------------------------------------------------------------------------------------------
# registry (models.py:289-322)
# ---------------------------------------------------------------------------------------------
def _warmup_only_process_fn(*a, **k):
    raise NotImplementedError("process_fn is used only by the warm-up trainer (data/process_fn.py), out of scope")


default_process_fn = _warmup_only_process_fn


def _hf(name):
    def get():
        import transformers
        return getattr(transformers, name)
    return get


class MSMarcoConfig:
    def __init__(self, name, model, process_fn=default_process_fn, use_mean=True, tokenizer_class=None,
                 config_class=None):
        self.name = name
        self.process_fn = process_fn
        self.model_class = model
        self.use_mean = use_mean
        self._tokenizer_class = tokenizer_class or _hf("RobertaTokenizer")
        self._config_class = config_class or _hf("RobertaConfig")

    @property
    def tokenizer_class(self):
        return self._tokenizer_class()

    @property
    def config_class(self):
        return self._config_class()


configs = [
    MSMarcoConfig(name="rdot_nll", model=RobertaDot_NLL_LN, use_mean=False),
    MSMarcoConfig(name="rdot_nll_multi_chunk", model=RobertaDot_CLF_ANN_NLL_MultiChunk, use_mean=False),
    MSMarcoConfig(name="dpr", model=BiEncoder, tokenizer_class=_hf("BertTokenizer"), config_class=_hf("BertConfig"),
                  use_mean=False),
    MSMarcoConfig(name="seeddot_nll", model=SEEDEncoderDot_NLL_LN, use_mean=False,
                  config_class=lambda: SEEDEncoderConfig),
]

MSMarcoConfigDict = {cfg.name: cfg for cfg in configs}
ALL_MODELS = ()
