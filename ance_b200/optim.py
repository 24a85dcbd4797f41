"""Lamb and AdamW on the sm_90a kernels: drop-ins for the reference trainers' `from utils.lamb import Lamb` and
`from transformers import AdamW` (transformers 2.3.0).

Lamb's update rule, per parameter p with gradient g of a group (lr, betas = (b1, b2), eps, weight_decay = wd):

    step += 1
    m <- b1 m + (1 - b1) g ;  v <- b2 v + (1 - b2) g^2            (no bias correction)
    u  = m / (sqrt(v) + eps) + wd p                              (p before this step's update; wd p only when wd != 0)
    w  = min(||p||, 10) ;  a = ||u|| ;  r = w / a, or 1 when w or a is 0
    p <- p - lr (1 if adam else r) u
    state: step, exp_avg = m, exp_avg_sq = v, weight_norm = w, adam_norm = a, trust_ratio = r (before the adam override)

`step()` runs it for every parameter of one device in one `ance_lamb_step` call (three kernels, per 512 tensors): no
host synchronisation, no torch kernels once every parameter has its state.  `weight_norm`, `adam_norm` and `trust_ratio`
are 0-d views into one [tensors, 3] device buffer the kernel writes; state dicts round-trip with the reference class's
in both directions.

AdamW's update rule, per parameter p with gradient g of a group (lr, betas = (b1, b2), eps, weight_decay = wd,
correct_bias):

    step += 1
    m <- b1 m + (1 - b1) g ;  v <- b2 v + (1 - b2) g^2
    step_size = lr sqrt(1 - b2^step) / (1 - b1^step) if correct_bias else lr      (in double, on the host)
    p <- p - step_size m / (sqrt(v) + eps)
    p <- p - lr wd p                                                             (the updated p; only when wd > 0)
    state: step (a Python int), exp_avg = m, exp_avg_sq = v

`step()` runs it for every parameter of one device in one `ance_adamw_step` call (one kernel, per 512 tensors).

Neither step synchronises with the host, and neither falls back to the CPU: parameters and gradients must be contiguous
fp32 CUDA tensors.
"""
from __future__ import annotations

import collections
import math

import numpy as np
import torch
from torch.autograd.graph import increment_version
from torch.optim import Optimizer

from . import _lib

MAX_TENSORS_PER_CALL = 512   # table capacity of ance_lamb_step and ance_adamw_step


def log_lamb_rs(optimizer: Optimizer, event_writer, token_count: int) -> None:
    """Histograms of the per-tensor weight_norm, adam_norm and trust_ratio of the last step (tensorboard `lamb/<key>`)."""
    results = collections.defaultdict(list)
    for group in optimizer.param_groups:
        for p in group["params"]:
            state = optimizer.state[p]
            for key in ("weight_norm", "adam_norm", "trust_ratio"):
                if key in state:
                    results[key].append(state[key])
    for key, values in results.items():
        event_writer.add_histogram(f"lamb/{key}", torch.tensor(values), token_count)


def _check(name: str, t: torch.Tensor, what: str, dev: torch.device) -> None:
    if t.layout is not torch.strided:
        raise _lib.AnceError(f"{name}: sparse {what} are not supported")
    if t.device != dev:
        raise _lib.AnceError(f"{name}: {what} on {t.device}; every parameter, gradient and state of one step must be "
                             f"on one CUDA device ({dev}) — there is no CPU fallback")
    if t.dtype is not torch.float32 or not t.is_contiguous():
        raise _lib.AnceError(f"{name}: {what} must be contiguous fp32 (got {t.dtype}, "
                             f"{'contiguous' if t.is_contiguous() else 'strided'})")


def _stepped(opt: Optimizer, name: str):
    """-> ([(group, p, grad, state)] of every parameter with a gradient, in group order, with its state created where it
    was missing (step 0, zero moments) and its step counted; the device they are on, or None).  Raises AnceError for what
    the kernels cannot take: a CPU parameter, non-fp32, strided or sparse tensors, more than one device, or a gradient or
    moment of another shape than its parameter."""
    items, dev = [], None
    for group in opt.param_groups:
        for p in group["params"]:
            g = p.grad
            if g is None:
                continue
            if dev is None:
                dev = p.device
                if dev.type != "cuda":
                    raise _lib.AnceError(f"{name}: parameter on {dev}; the step runs on an sm_90 GPU only (no CPU "
                                         "fallback): move the model to a CUDA device")
            _check(name, p, "parameters", dev)
            _check(name, g, "gradients", dev)
            if g.shape != p.shape:
                raise _lib.AnceError(f"{name}: gradient of shape {tuple(g.shape)} for a parameter of shape "
                                     f"{tuple(p.shape)}")
            state = opt.state[p]
            if len(state) == 0:
                state["step"] = 0
                state["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
            m, v = state["exp_avg"], state["exp_avg_sq"]
            _check(name, m, "exp_avg states", dev)
            _check(name, v, "exp_avg_sq states", dev)
            if m.shape != p.shape or v.shape != p.shape:
                raise _lib.AnceError(f"{name}: exp_avg / exp_avg_sq state of another shape than its parameter")
            state["step"] += 1
            items.append((group, p, g, state))
    return items, dev


def _tables(items):
    """The device pointers [4, n] (p, g, exp_avg, exp_avg_sq) and element counts [n] of the kernels' tensor table."""
    ptrs = np.array([[t.data_ptr() for t in ts] for ts in
                     zip(*((p, g, st["exp_avg"], st["exp_avg_sq"]) for _, p, g, st in items))], dtype=np.uint64)
    return ptrs, np.array([p.numel() for _, p, _, _ in items], dtype=np.int64)


class Lamb(Optimizer):
    r"""Lamb (You et al., "Large Batch Optimization for Deep Learning: Training BERT in 76 minutes",
    arXiv:1904.00962, v3 without bias correction), as the reference trainer configures it.

    Arguments:
        params: iterable of parameters or dicts defining parameter groups
        lr: learning rate (default 1e-3)
        betas: coefficients of the running averages of the gradient and its square (default (0.9, 0.999))
        eps: added to the denominator (default 1e-6)
        weight_decay: decoupled weight decay added to the Adam step before the trust ratio (default 0)
        adam: use trust ratio 1 (plain Adam without bias correction), for comparison
    """

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0, adam=False):
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: {}".format(lr))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: {}".format(eps))
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError("Invalid beta parameter at index 0: {}".format(betas[0]))
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid beta parameter at index 1: {}".format(betas[1]))
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        self.adam = adam
        super().__init__(params, defaults)
        self._norms_key = None   # ids of the parameters the norms buffer's rows belong to
        self._norms = None

    def __setstate__(self, state):
        super().__setstate__(state)
        self._norms_key = None
        self._norms = None

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._norms_key = None   # the loaded weight_norm / adam_norm / trust_ratio are not views of our buffer
        self._norms = None

    def step(self, closure=None):
        """One Lamb step over every parameter that has a gradient.  Returns the closure's loss (None without one)."""
        loss = None
        if closure is not None:
            loss = closure()
        items, dev = _stepped(self, "Lamb")
        if not items:
            return loss
        params = [p for _, p, _, _ in items]
        hyp = np.array([(float(gr["lr"]), float(gr["betas"][0]), float(gr["betas"][1]), float(gr["eps"]),
                         float(gr["weight_decay"])) for gr, _, _, _ in items], dtype=np.float64)
        ptrs, numel = _tables(items)
        with torch.cuda.device(dev):
            norms = self._norms_for(params, dev)
            lib, stream = _lib.load(), torch.cuda.current_stream(dev).cuda_stream
            n = len(params)
            for i0 in range(0, n, MAX_TENSORS_PER_CALL):
                k = min(MAX_TENSORS_PER_CALL, n - i0)
                _lib.check(lib.ance_lamb_step(k, ptrs[0, i0:].ctypes.data, ptrs[1, i0:].ctypes.data,
                                              ptrs[2, i0:].ctypes.data, ptrs[3, i0:].ctypes.data,
                                              numel[i0:].ctypes.data, hyp[i0:].ctypes.data, 1 if self.adam else 0,
                                              norms[i0].data_ptr(), stream))
        increment_version(params)   # written in place, as p.add_ would: cached copies of the weights see the change
        return loss

    def _norms_for(self, params, dev) -> torch.Tensor:
        """The [n, 3] (w, a, r) buffer of this parameter list; its rows are the parameters' weight_norm, adam_norm and
        trust_ratio state.  Rebuilt (no kernel: torch.empty and views) when the list changes."""
        key = [id(p) for p in params]
        if key != self._norms_key or self._norms.device != dev:
            buf = torch.empty((len(params), 3), dtype=torch.float32, device=dev)
            for i, p in enumerate(params):
                state = self.state[p]
                state["weight_norm"], state["adam_norm"], state["trust_ratio"] = buf[i, 0], buf[i, 1], buf[i, 2]
            self._norms, self._norms_key = buf, key
        return self._norms


class AdamW(Optimizer):
    r"""Adam with decoupled weight decay (Loshchilov & Hutter, "Decoupled Weight Decay Regularization",
    arXiv:1711.05101), transformers 2.3.0's AdamW as the reference trainers build it (`--optimizer adamW`).

    It is not torch.optim.AdamW: eps is added to sqrt(v) before any bias correction, the bias correction goes into the
    step size, and the weight decay is applied after the Adam update, to the updated parameter, and only when
    weight_decay > 0.

    Arguments:
        params: iterable of parameters or dicts defining parameter groups
        lr: learning rate (default 1e-3)
        betas: coefficients of the running averages of the gradient and its square (default (0.9, 0.999))
        eps: added to the denominator (default 1e-6)
        weight_decay: decoupled weight decay, applied when > 0 (default 0)
        correct_bias: fold Adam's bias correction into the step size (default True)
    """

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True):
        if lr < 0.0:
            raise ValueError("Invalid learning rate: {} - should be >= 0.0".format(lr))
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError("Invalid beta parameter: {} - should be in [0.0, 1.0[".format(betas[0]))
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid beta parameter: {} - should be in [0.0, 1.0[".format(betas[1]))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: {} - should be >= 0.0".format(eps))
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, correct_bias=correct_bias)
        super().__init__(params, defaults)

    def step(self, closure=None):
        """One AdamW step over every parameter that has a gradient.  Returns the closure's loss (None without one)."""
        loss = None
        if closure is not None:
            loss = closure()
        items, dev = _stepped(self, "AdamW")
        if not items:
            return loss
        hyper = []
        for group, _, _, state in items:
            beta1, beta2 = group["betas"]
            lr, step = float(group["lr"]), state["step"]
            step_size = lr
            if group["correct_bias"]:
                step_size = lr * math.sqrt(1.0 - beta2 ** step) / (1.0 - beta1 ** step)
            hyper.append((step_size, float(beta1), float(beta2), float(group["eps"]),
                          lr * float(group["weight_decay"])))
        hyp = np.array(hyper, dtype=np.float64)
        ptrs, numel = _tables(items)
        params = [p for _, p, _, _ in items]
        with torch.cuda.device(dev):
            lib, stream = _lib.load(), torch.cuda.current_stream(dev).cuda_stream
            n = len(params)
            for i0 in range(0, n, MAX_TENSORS_PER_CALL):
                k = min(MAX_TENSORS_PER_CALL, n - i0)
                _lib.check(lib.ance_adamw_step(k, ptrs[0, i0:].ctypes.data, ptrs[1, i0:].ctypes.data,
                                               ptrs[2, i0:].ctypes.data, ptrs[3, i0:].ctypes.data,
                                               numel[i0:].ctypes.data, hyp[i0:].ctypes.data, stream))
        increment_version(params)   # written in place, as p.add_ would: cached copies of the weights see the change
        return loss
