"""Two restatements of the reference trainer's Lamb step (utils/lamb.py), the yardsticks of ance_b200.optim.Lamb.

  lamb_step_fp64  one step of one tensor in float64 from fp32 inputs: the per-element truth the kernel is held to.
  EagerLamb       a torch.optim.Optimizer with the reference's state layout and its fp32 operation sequence, one eager
                  pass per tensor with the reference's host synchronisations (the truth value of `w == 0 or a == 0`, a
                  0-d CUDA tensor as the update's alpha).  On CPU it reproduces the reference bit for bit; it is the
                  baseline tools/bench_optim.py times and the other side of the state-dict interop tests.

The rule: m <- b1 m + (1 - b1) g; v <- b2 v + (1 - b2) g^2; u = m / (sqrt(v) + eps) (+ wd p when wd != 0);
w = clamp(||p||, 0, 10); a = ||u||; r = w / a unless w or a is 0 (then 1); p <- p - lr (adam ? 1 : r) u.
"""
from __future__ import annotations

import torch
from torch.optim import Optimizer


def lamb_step_fp64(p, g, m, v, lr, beta1, beta2, eps, weight_decay=0.0, adam=False):
    """torch tensors (any float dtype, any device) -> float64 (p, m, v, w, a, r) after one step; w, a, r python floats."""
    p, g, m, v = (x.double() for x in (p, g, m, v))
    m = beta1 * m + (1.0 - beta1) * g
    v = beta2 * v + (1.0 - beta2) * g * g
    u = m / (v.sqrt() + eps)
    if weight_decay != 0:
        u = u + weight_decay * p
    norm_p = float(p.square().sum().sqrt())
    w = 10.0 if norm_p > 10.0 else norm_p   # clamp(0, 10); NaN stays NaN
    a = float(u.square().sum().sqrt())
    r = 1.0 if (w == 0 or a == 0) else w / a
    p = p - lr * (1.0 if adam else r) * u
    return p, m, v, w, a, r


def lamb_step_bounds(p, g, m, v, out, lr, beta1, beta2, eps, weight_decay=0.0, adam=False):
    """Per-element bounds (tol_p, tol_m, tol_v), float64 tensors, for an fp32 implementation of one step against
    lamb_step_fp64's `out`: 2 ulp of the operands' scale for m (b1 m and (1 - b1) g may cancel) and v, the resulting
    error of u = m / (sqrt(v) + eps) carried through lr r, plus 2 ulp(p) and 1e-5 |dp| for the fp32 norms behind r."""
    e = 2.0 ** -23   # ulp(x) <= e |x| for normal fp32 x
    p, g, m, v = (x.double() for x in (p, g, m, v))
    p1, m1, v1, _, _, r = out
    tol_m = 2 * e * (beta1 * m.abs() + (1.0 - beta1) * g.abs())
    tol_v = 2 * e * v1
    den = v1.sqrt() + eps
    u = m1 / den + (weight_decay * p if weight_decay != 0 else 0.0)
    tol_u = tol_m / den + 4 * e * (m1 / den).abs() + 2 * e * u.abs()
    tol_p = 2 * e * p1.abs() + lr * (1.0 if adam else r) * tol_u + 1e-5 * (p1 - p).abs()
    return tol_p, tol_m, tol_v


class EagerLamb(Optimizer):
    """The reference's Lamb, op for op in fp32 (current torch spellings of the same in-place calls)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0, adam=False):
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: {}".format(lr))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: {}".format(eps))
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError("Invalid beta parameter at index 0: {}".format(betas[0]))
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid beta parameter at index 1: {}".format(betas[1]))
        self.adam = adam
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    def step(self, closure=None):
        loss = closure() if closure is not None else None
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                grad = p.grad.data
                if grad.is_sparse:
                    raise RuntimeError("Lamb does not support sparse gradients")
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    state["exp_avg"] = torch.zeros_like(p.data)
                    state["exp_avg_sq"] = torch.zeros_like(p.data)
                exp_avg, exp_avg_sq = state["exp_avg"], state["exp_avg_sq"]
                state["step"] += 1
                exp_avg.mul_(beta1).add_(grad, alpha=1 - beta1)
                exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
                weight_norm = p.data.pow(2).sum().sqrt().clamp(0, 10)
                adam_step = exp_avg / exp_avg_sq.sqrt().add(group["eps"])
                if group["weight_decay"] != 0:
                    adam_step.add_(p.data, alpha=group["weight_decay"])
                adam_norm = adam_step.pow(2).sum().sqrt()
                if weight_norm == 0 or adam_norm == 0:     # two host synchronisations
                    trust_ratio = 1
                else:
                    trust_ratio = weight_norm / adam_norm
                state["weight_norm"] = weight_norm
                state["adam_norm"] = adam_norm
                state["trust_ratio"] = trust_ratio
                if self.adam:
                    trust_ratio = 1
                p.data.add_(adam_step, alpha=-group["lr"] * trust_ratio)   # a 0-d tensor alpha: a third one
        return loss
