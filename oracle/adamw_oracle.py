"""Two restatements of transformers 2.3.0's AdamW step (the reference trainers' `--optimizer adamW`), the yardsticks of
ance_b200.optim.AdamW.  transformers 2.3.0 is not vendored in the reference, so the rule is restated here from its
AdamW.step; tests/test_adamw_cpu.py ties it to code the reference ships (utils/lamb.py with adam=True is the same step
without bias correction and weight decay).

  adamw_step_fp64   one step of one tensor in float64 from fp32 inputs: the per-element truth the kernel is held to.
  adamw_step_bounds per-element tolerances for an fp32 implementation of that step.
  EagerAdamW        a torch.optim.Optimizer with the reference's state layout (int step, exp_avg, exp_avg_sq) and its fp32
                    operation sequence, one eager pass per tensor: the baseline tools/bench_optim.py times and the other
                    side of the state-dict interop tests.

The rule: step += 1; m <- b1 m + (1 - b1) g; v <- b2 v + (1 - b2) g^2; step_size = lr sqrt(1 - b2^step) / (1 - b1^step)
with correct_bias (lr without), in Python double; p <- p - step_size m / (sqrt(v) + eps); then, only when
weight_decay > 0, p <- p - lr weight_decay p on the updated p.
"""
from __future__ import annotations

import math

import torch
from torch.optim import Optimizer


def _step_size(lr, beta1, beta2, step, correct_bias):
    if not correct_bias:
        return lr
    return lr * math.sqrt(1.0 - beta2 ** step) / (1.0 - beta1 ** step)


def adamw_step_fp64(p, g, m, v, step, lr, beta1, beta2, eps, weight_decay=0.0, correct_bias=True):
    """torch tensors (any float dtype, any device) and the step count after this step -> float64 (p, m, v)."""
    p, g, m, v = (x.double() for x in (p, g, m, v))
    m = beta1 * m + (1.0 - beta1) * g
    v = beta2 * v + (1.0 - beta2) * g * g
    p = p - _step_size(lr, beta1, beta2, step, correct_bias) * (m / (v.sqrt() + eps))
    if weight_decay > 0.0:
        p = p - lr * weight_decay * p
    return p, m, v


def adamw_step_bounds(p, g, m, v, out, step, lr, beta1, beta2, eps, weight_decay=0.0, correct_bias=True):
    """Per-element bounds (tol_p, tol_m, tol_v), float64 tensors, for an fp32 implementation of one step against
    adamw_step_fp64's `out`, derived as lamb_step_bounds: 2 ulp of the operands' scale for m (b1 m and (1 - b1) g may
    cancel) and v; the error of q = m / (sqrt(v) + eps) that follows (that of m, plus 4 ulp for v, the square root, the
    sum and the quotient); q's error and one ulp of step_size q carried into p, plus 2 ulp(p); the decay's factor
    (1 - lr wd) applied to all of that, plus one ulp of lr wd p."""
    e = 2.0 ** -23   # ulp(x) <= e |x| for normal fp32 x
    p, g, m, v = (x.double() for x in (p, g, m, v))
    p1, m1, v1 = out
    tol_m = 2 * e * (beta1 * m.abs() + (1.0 - beta1) * g.abs())
    tol_v = 2 * e * v1
    q = m1 / (v1.sqrt() + eps)
    tol_q = tol_m / (v1.sqrt() + eps) + 4 * e * q.abs()
    s = _step_size(lr, beta1, beta2, step, correct_bias)
    tol_p = s * (tol_q + e * q.abs())
    if weight_decay > 0.0:
        d = lr * weight_decay
        tol_p = tol_p * (1.0 + d) + e * d * (p1.abs() / max(1.0 - d, 1e-30))
    return tol_p + 2 * e * p1.abs(), tol_m, tol_v


class EagerAdamW(Optimizer):
    """transformers 2.3.0's AdamW, op for op in fp32 (current torch spellings of the same in-place calls)."""

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
        loss = closure() if closure is not None else None
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                grad = p.grad.data
                if grad.is_sparse:
                    raise RuntimeError("Adam does not support sparse gradients, please consider SparseAdam instead")
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    state["exp_avg"] = torch.zeros_like(p.data)
                    state["exp_avg_sq"] = torch.zeros_like(p.data)
                exp_avg, exp_avg_sq = state["exp_avg"], state["exp_avg_sq"]
                beta1, beta2 = group["betas"]
                state["step"] += 1
                exp_avg.mul_(beta1).add_(grad, alpha=1.0 - beta1)
                exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1.0 - beta2)
                denom = exp_avg_sq.sqrt().add_(group["eps"])
                step_size = group["lr"]
                if group["correct_bias"]:
                    bias_correction1 = 1.0 - beta1 ** state["step"]
                    bias_correction2 = 1.0 - beta2 ** state["step"]
                    step_size = step_size * math.sqrt(bias_correction2) / bias_correction1
                p.data.addcdiv_(exp_avg, denom, value=-step_size)
                if group["weight_decay"] > 0.0:
                    p.data.add_(p.data, alpha=-group["lr"] * group["weight_decay"])
        return loss
