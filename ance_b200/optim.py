"""Lamb on the sm_90a kernels: a drop-in for the reference trainer's `from utils.lamb import Lamb`.

The update rule, per parameter p with gradient g of a group (lr, betas = (b1, b2), eps, weight_decay = wd):

    step += 1
    m <- b1 m + (1 - b1) g ;  v <- b2 v + (1 - b2) g^2            (no bias correction)
    u  = m / (sqrt(v) + eps) + wd p                              (p before this step's update; wd p only when wd != 0)
    w  = min(||p||, 10) ;  a = ||u|| ;  r = w / a, or 1 when w or a is 0
    p <- p - lr (1 if adam else r) u
    state: step, exp_avg = m, exp_avg_sq = v, weight_norm = w, adam_norm = a, trust_ratio = r (before the adam override)

`step()` runs it for every parameter of one device in one `ance_lamb_step` call (three kernels, per 512 tensors): no
host synchronisation, no torch kernels once every parameter has its state.  `weight_norm`, `adam_norm` and `trust_ratio`
are 0-d views into one [tensors, 3] device buffer the kernel writes; state dicts round-trip with the reference class's
in both directions.  There is no CPU fallback: parameters and gradients must be contiguous fp32 CUDA tensors.
"""
from __future__ import annotations

import collections

import numpy as np
import torch
from torch.autograd.graph import increment_version
from torch.optim import Optimizer

from . import _lib

MAX_TENSORS_PER_CALL = 512   # ance_lamb_step's table capacity


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


def _check(t: torch.Tensor, what: str, dev: torch.device) -> None:
    if t.layout is not torch.strided:
        raise _lib.AnceError(f"Lamb: sparse {what} are not supported")
    if t.device != dev:
        raise _lib.AnceError(f"Lamb: {what} on {t.device}; every parameter, gradient and state of one step must be on "
                             f"one CUDA device ({dev}) — there is no CPU fallback")
    if t.dtype is not torch.float32 or not t.is_contiguous():
        raise _lib.AnceError(f"Lamb: {what} must be contiguous fp32 (got {t.dtype}, "
                             f"{'contiguous' if t.is_contiguous() else 'strided'})")


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
        params, grads, exp_avgs, exp_avg_sqs, hyper = [], [], [], [], []
        dev = None
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            hp = (float(group["lr"]), float(beta1), float(beta2), float(group["eps"]), float(group["weight_decay"]))
            for p in group["params"]:
                g = p.grad
                if g is None:
                    continue
                if dev is None:
                    dev = p.device
                    if dev.type != "cuda":
                        raise _lib.AnceError(f"Lamb: parameter on {dev}; the step runs on an sm_90 GPU only (no CPU "
                                             "fallback): move the model to a CUDA device")
                _check(p, "parameters", dev)
                _check(g, "gradients", dev)
                if g.shape != p.shape:
                    raise _lib.AnceError(f"Lamb: gradient of shape {tuple(g.shape)} for a parameter of shape "
                                         f"{tuple(p.shape)}")
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                m, v = state["exp_avg"], state["exp_avg_sq"]
                _check(m, "exp_avg states", dev)
                _check(v, "exp_avg_sq states", dev)
                if m.shape != p.shape or v.shape != p.shape:
                    raise _lib.AnceError("Lamb: exp_avg / exp_avg_sq state of another shape than its parameter")
                state["step"] += 1
                params.append(p)
                grads.append(g)
                exp_avgs.append(m)
                exp_avg_sqs.append(v)
                hyper.append(hp)
        if not params:
            return loss
        with torch.cuda.device(dev):
            norms = self._norms_for(params, dev)
            lib, stream = _lib.load(), torch.cuda.current_stream(dev).cuda_stream
            n = len(params)
            ptrs = np.array([[t.data_ptr() for t in ts] for ts in (params, grads, exp_avgs, exp_avg_sqs)],
                            dtype=np.uint64)
            numel = np.array([p.numel() for p in params], dtype=np.int64)
            hyp = np.ascontiguousarray(hyper, dtype=np.float64)
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
