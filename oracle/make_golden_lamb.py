"""Generate tests/golden/lamb_steps.npz by running the REFERENCE's own Lamb (utils/lamb.py) on CPU.

Run in the build container only (the GPU machine has no reference checkout):

    python oracle/make_golden_lamb.py

What is pinned (LAMB_SPEC below): seeded small fp32 tensors in two groups (group 0: lr 1e-2, eps 1e-8, no weight decay;
group 1: lr 3e-3, the class's eps 1e-6, weight decay 1e-2) covering a zero bias (w = 0 on the first step), a matrix with
||p|| > 10 (w clamped), a tensor whose gradient is always 0 from zero state (a = 0), a parameter whose .grad stays None,
a one-element tensor and odd sizes.  STEPS steps with fresh seeded gradients, once with adam=False and once with
adam=True.  Stored: every tensor's initial value `<name>/p0`, its gradients `<name>/g` [STEPS, ...], and per run
(`lamb`, `adam`) `<run>/<name>/{p,m,v}` [STEPS, ...] and `<run>/<name>/war` [STEPS, 3] (weight_norm, adam_norm,
trust_ratio) after every step; `meta` is the JSON of LAMB_SPEC, LAMB_GROUPS and STEPS.
"""
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
GOLD = os.path.join(ROOT, "tests", "golden")

STEPS = 20
# name -> (shape, group, init std (0: zeros), gradient std (0: always zero, None: .grad stays None))
LAMB_SPEC = {
    "bias_zero": ((17,), 0, 0.0, 1e-2),
    "big_matrix": ((12, 14), 0, 1.0, 3e-3),
    "zero_grad": ((13,), 0, 0.02, 0.0),
    "no_grad": ((5,), 0, 0.02, None),
    "odd": ((61,), 1, 0.02, 1e-2),
    "one": ((1,), 1, 0.5, 1e-1),
    "matrix_wd": ((5, 7), 1, 0.5, 2e-2),
}
LAMB_GROUPS = ({"lr": 1e-2, "eps": 1e-8}, {"lr": 3e-3, "weight_decay": 1e-2})


def lamb_tensors():
    """The seeded initial tensors and per-step gradients of LAMB_SPEC -> ({name: p0}, {name: [STEPS grads] or None})."""
    p0, grads = {}, {}
    for i, (name, (shape, _, std, gstd)) in enumerate(LAMB_SPEC.items()):
        gen = torch.Generator().manual_seed(1000 + i)
        p0[name] = torch.randn(shape, generator=gen) * std if std else torch.zeros(shape)
        if gstd is None:
            grads[name] = None
        else:
            grads[name] = torch.stack([torch.randn(shape, generator=gen) * gstd if gstd else torch.zeros(shape)
                                       for _ in range(STEPS)])
    return p0, grads


def golden_lamb():
    sys.path.append(REF)
    sys.modules.setdefault("tensorboardX", types.ModuleType("tensorboardX"))
    sys.modules["tensorboardX"].SummaryWriter = object
    from utils.lamb import Lamb   # the reference's own class

    p0, grads = lamb_tensors()
    out = {"meta": np.array(json.dumps({"spec": {k: [list(v[0]), v[1], v[2], v[3]] for k, v in LAMB_SPEC.items()},
                                        "groups": LAMB_GROUPS, "steps": STEPS}))}
    for name in LAMB_SPEC:
        out[f"{name}/p0"] = p0[name].numpy()
        if grads[name] is not None:
            out[f"{name}/g"] = grads[name].numpy()
    for run, adam in (("lamb", False), ("adam", True)):
        params = {k: torch.nn.Parameter(v.clone()) for k, v in p0.items()}
        groups = [dict(LAMB_GROUPS[gi], params=[params[k] for k, v in LAMB_SPEC.items() if v[1] == gi])
                  for gi in range(len(LAMB_GROUPS))]
        opt = Lamb(groups, adam=adam)
        rec = {k: {"p": [], "m": [], "v": [], "war": []} for k in LAMB_SPEC if grads[k] is not None}
        for s in range(STEPS):
            for k, p in params.items():
                p.grad = None if grads[k] is None else grads[k][s].clone()
            opt.step()
            for k, r in rec.items():
                st = opt.state[params[k]]
                r["p"].append(params[k].detach().numpy().copy())
                r["m"].append(st["exp_avg"].numpy().copy())
                r["v"].append(st["exp_avg_sq"].numpy().copy())
                r["war"].append([float(st[x]) for x in ("weight_norm", "adam_norm", "trust_ratio")])
        assert "no_grad" not in opt.state or not opt.state[params["no_grad"]]
        for k, r in rec.items():
            for f in ("p", "m", "v"):
                out[f"{run}/{k}/{f}"] = np.stack(r[f]).astype(np.float32)
            out[f"{run}/{k}/war"] = np.array(r["war"], dtype=np.float32)
    path = os.path.join(GOLD, "lamb_steps.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    golden_lamb()
