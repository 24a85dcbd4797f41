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
Training: after ``model.set_trainable(True)`` (rdot_nll, inputs of up to 128 tokens) ``query_emb`` / ``body_emb`` /
``forward()`` build an autograd graph whose backward runs the encoder's own backward kernels, so ``loss.backward()``
fills the parameters' ``.grad``; by default the outputs carry no graph.
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


def _dev_ptr(t: torch.Tensor):
    return C.cast(C.c_void_p(t.data_ptr()), C.POINTER(C.c_float))


class _CudaEncoder:
    """Owns one ance_encoder handle built from a backbone's current parameters."""

    def __init__(self, backbone: nn.Module, arch: int, heads: int, pad_id: int, head: Optional[tuple],
                 max_tokens: int, device: torch.device, operand: str = "fp16"):
        lib = _lib.load()
        self.lib = lib
        self.device = device
        emb = backbone.embeddings
        H = emb.word_embeddings.weight.shape[1]
        layers = list(backbone.encoder.layer)
        cfg = _lib.EncoderConfig()
        cfg.arch = arch
        cfg.n_layer = len(layers)
        cfg.hidden = H
        cfg.heads = heads
        cfg.ffn = layers[0].intermediate.dense.weight.shape[0]
        cfg.vocab = emb.word_embeddings.weight.shape[0]
        cfg.max_pos = emb.position_embeddings.weight.shape[0]
        cfg.type_vocab = emb.token_type_embeddings.weight.shape[0]
        cfg.pad_id = pad_id
        cfg.ln_eps = float(emb.LayerNorm.eps)
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
        w, lw = _fill(_lib.EncoderWeights, _lib.LayerWeights, _param_groups(backbone, head), fp)
        self.hidden_size = H
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

    def forward_train(self, ids: torch.Tensor, lens: Optional[torch.Tensor], mask: Optional[torch.Tensor]):
        """forward() of a whole [B, L <= 128] batch that also keeps what the backward needs.  -> (out fp32 [B, H],
        workspace tensor for backward())."""
        B, L = ids.shape
        n = C.c_size_t()
        _lib.check(self.lib.ance_encoder_train_workspace(self.h, B, L, C.byref(n)))
        ws = torch.empty(n.value, dtype=torch.uint8, device=ids.device)
        out = torch.empty((B, self.hidden_size), dtype=torch.float32, device=ids.device)
        with torch.cuda.device(ids.device):
            _lib.check(self.lib.ance_encoder_forward_train(
                self.h, ids.data_ptr(), None if lens is None else lens.data_ptr(),
                None if mask is None else mask.data_ptr(), B, L, ws.data_ptr(), out.data_ptr(), _lib.current_stream()))
        return out, ws

    def backward(self, d_out: torch.Tensor, ws: torch.Tensor, grads) -> None:
        """Gradients of sum(d_out * out) for the forward_train that filled `ws`, written into `grads` (fp32 tensors
        grouped as _param_groups)."""
        w, lw = _fill(_lib.EncoderGrads, _lib.LayerGrads, grads, _dev_ptr)
        with torch.cuda.device(d_out.device):
            _lib.check(self.lib.ance_encoder_backward(self.h, d_out.data_ptr(), ws.data_ptr(), C.byref(w),
                                                      _lib.current_stream()))


class _TrainableEncode(torch.autograd.Function):
    """Embeddings [B, H] of a dense batch as a function of the encoder's parameters (the `params` inputs, in
    _param_groups order), so that their .grad accumulates and DDP's hooks fire."""

    @staticmethod
    def forward(ctx, enc, n_layer, ids, lens, mask, *params):
        out, ws = enc.forward_train(ids, lens, mask)
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
        return (None, None, None, None, None, *flat)


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

    #: set_trainable(True): embeddings computed while grad is enabled carry an autograd graph (dense, L <= 128)
    _trainable = False

    def set_trainable(self, on: bool = True):
        """Opt in to gradients: while torch grad mode is on, query_emb / body_emb / encode_lens (dense batches of up to
        128 tokens) and the triplet forward() return tensors whose backward runs the encoder's backward kernels; the
        other encode paths raise instead of returning detached results.  Off by default."""
        self._trainable = bool(on)
        return self

    def _grad_path(self) -> bool:
        return self._trainable and torch.is_grad_enabled()

    def _refuse_grad(self, what: str) -> None:
        if self._grad_path():
            raise _lib.AnceError(f"{what} has no backward: trainable encoders take dense batches of up to 128 tokens "
                                 "through query_emb / body_emb / encode_lens (or run this under torch.no_grad())")

    def _train_emb(self, enc, backbone, head, ids, lens, mask):
        B, L = ids.shape
        if L > 128:
            raise _lib.AnceError(f"inputs of {L} tokens have no backward: the trainable encoder covers up to 128 tokens "
                                 "(run longer inputs under torch.no_grad())")
        if B * L > enc.max_tokens:
            raise _lib.AnceError(f"a trainable batch of {B} x {L} tokens exceeds max_tokens {enc.max_tokens}")
        # The device weights are refreshed from the parameters before every training forward, whatever their `_version`
        # says: optimizers that write through `p.data` (the reference trainer's Lamb, transformers' AdamW) do not bump it.
        if not enc.update_weights(backbone, head):
            raise _lib.AnceError("a trainable encoder needs contiguous fp32 parameters on the inputs' device")
        embs, layers, hd = _param_groups(backbone, head)
        params = embs + [t for l in layers for t in l] + hd
        return _TrainableEncode.apply(enc, len(layers), ids, lens, mask, *params)

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
    # autograd graph through the encoder's backward kernels (inputs of up to 128 tokens); otherwise it is computed
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
        model = cls(config)
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
        model.load_state_dict({k: sd[k] for k in own}, strict=True)  # classifier.*, pooler.*: unused (SURVEY §8 a2)
        model.eval()
        return model

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
                           out: Optional[torch.Tensor] = None, align: int = 1) -> torch.Tensor:
        """encode_lens at the cost of the REAL tokens only, for any L <= 512 (lengths in [1, L]).  align = 16: bit-identical
        to encode_lens at the same L, whatever else is in the batch; align = 1: densest packing, equal up to fp32
        summation order.  L <= 128 is encode_lens_varlen."""
        self._refuse_grad("encode_lens_packed")
        return self._encoder(ids_i32.device).forward_packed(ids_i32.contiguous(), lens_i32.contiguous(), lens_host, out=out,
                                                            align=align)

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
        self._refuse_grad("the multi-chunk body_emb")
        batchS, full_length = input_ids.shape
        chunk_factor = full_length // self.base_len
        if chunk_factor == 0 or full_length % chunk_factor != 0:
            raise ValueError(f"document length {full_length} is not a multiple of base_len {self.base_len}")
        seq = full_length // chunk_factor
        ids, mask = self._prep(input_ids.reshape(batchS * chunk_factor, seq),
                               attention_mask.reshape(batchS * chunk_factor, seq))
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

    def set_trainable(self, on: bool = True):
        if on:
            raise NotImplementedError("the DPR BiEncoder has no backward in ance_b200 (rdot_nll only)")
        return super().set_trainable(False)

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
        return enc.forward(ids, None, mask)

    def query_emb(self, input_ids, attention_mask):
        return self._emb("question", self.question_model, input_ids, attention_mask)

    def body_emb(self, input_ids, attention_mask):
        return self._emb("ctx", self.ctx_model, input_ids, attention_mask)

    def _emb_packed(self, name, backbone, input_ids, align, ids_host):
        """Same result as _emb(..., input_ids != 0) (DPR_data.py:283 mask) at the cost of the real tokens: rows whose
        nonzero ids form a non-empty prefix go through the packed forward, the others through the dense one.  The lengths
        are read from `ids_host` (the host copy of input_ids; copied back when not given)."""
        if input_ids.device.type != "cuda":
            raise _lib.AnceError("ance_b200 models run on an sm_90 GPU only (no CPU fallback)")
        ids = input_ids.to(torch.int32).contiguous()
        B, L = ids.shape
        nz = (ids_host if ids_host is not None else input_ids.cpu()).reshape(B, L) != 0
        lens = nz.sum(dim=1)
        ok = (nz == (torch.arange(L)[None, :] < lens[:, None])).all(dim=1) & (lens > 0)
        enc = self._enc_for(name, backbone, _lib.ANCE_ARCH_BERT, self.dims.num_attention_heads, 0, None, ids.device)
        lens32 = lens.to(torch.int32)
        if bool(ok.all()):
            return enc.forward_packed(ids, lens32.to(ids.device), lens32, align=align)
        out = torch.empty((B, self.dims.hidden_size), dtype=torch.float32, device=ids.device)
        sel, rest = torch.nonzero(ok).flatten(), torch.nonzero(~ok).flatten()
        if sel.numel():
            sd = sel.to(ids.device)
            out[sd] = enc.forward_packed(ids[sd].contiguous(), lens32[sel].to(ids.device), lens32[sel].contiguous(),
                                         align=align)
        rd = rest.to(ids.device)
        out[rd] = enc.forward(ids[rd].contiguous(), None, (ids[rd] != 0).to(torch.uint8).contiguous())
        return out

    def query_emb_packed(self, input_ids, align: int = 1, ids_host: Optional[torch.Tensor] = None):
        """query_emb(input_ids, input_ids != 0) computing the real tokens only (align: see encode_lens_packed)."""
        return self._emb_packed("question", self.question_model, input_ids, align, ids_host)

    def body_emb_packed(self, input_ids, align: int = 1, ids_host: Optional[torch.Tensor] = None):
        """body_emb(input_ids, input_ids != 0) computing the real tokens only (align: see encode_lens_packed)."""
        return self._emb_packed("ctx", self.ctx_model, input_ids, align, ids_host)

    @torch.no_grad()
    def forward(self, query_ids, attention_mask_q, input_ids_a=None, attention_mask_a=None, input_ids_b=None,
                attention_mask_b=None):
        """model/models.py:253-266 (evaluation only, no autograd): (q, a) embeddings, or `(loss,)` for triplets."""
        q_embs = self.query_emb(query_ids, attention_mask_q)
        a_embs = self.body_emb(input_ids_a, attention_mask_a)
        if input_ids_b is None:
            return (q_embs, a_embs)
        b_embs = self.body_emb(input_ids_b, attention_mask_b)
        logit_matrix = torch.stack([(q_embs * a_embs).sum(-1), (q_embs * b_embs).sum(-1)], dim=1)
        return ((-torch.log_softmax(logit_matrix, dim=1)[:, 0]).mean(),)


def _reference_seed_class():
    """The reference's own stock-PyTorch class, when the reference repository is importable (its directory on sys.path,
    as its scripts arrange with `sys.path += ['../']`)."""
    try:
        from model.models import SEEDEncoderDot_NLL_LN as ref_cls   # /root/reference-style checkout
        return ref_cls
    except Exception as e:  # ImportError, or the reference's own third-party imports failing
        raise NotImplementedError(
            "seeddot_nll (SEED-Encoder, model/models.py:201-221) has no sm_90a kernels in ance_b200 — its backbone is a "
            "vendored fairseq-style model outside the ANN-refresh scope (SURVEY.md par. 2.1 row 8) — and the reference's "
            "stock module could not be imported to fall back to ({}: {}).  Put the reference checkout on sys.path to run "
            "seeddot_nll through its own PyTorch code.".format(type(e).__name__, e)) from e


class SEEDEncoderDot_NLL_LN:
    """model/models.py:201-221 (`seeddot_nll`).  The registry name resolves; construction / from_pretrained FALL BACK to
    the reference's stock PyTorch module (SURVEY.md par. 2.1 row 8): the object returned is the reference's class, so
    `query_emb` / `body_emb` behave exactly as upstream (no GPU acceleration)."""

    def __new__(cls, *a, **k):
        return _reference_seed_class()(*a, **k)

    @classmethod
    def from_pretrained(cls, *a, **k):
        return _reference_seed_class().from_pretrained(*a, **k)


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
    MSMarcoConfig(name="seeddot_nll", model=SEEDEncoderDot_NLL_LN, use_mean=False),
]

MSMarcoConfigDict = {cfg.name: cfg for cfg in configs}
ALL_MODELS = ()
