"""AdamW without a GPU: the constructor's checks and defaults, the refusal of CPU tensors, the C entry point's argument
errors, the eager restatement (oracle/adamw_oracle.py) against its fp64 twin, the eager restatement against the
reference's own code (utils/lamb.py with adam=True is AdamW without bias correction and weight decay; its trajectory is
tests/golden/lamb_steps.npz's `adam` run), and state dicts in the reference's layout."""
import ctypes as C
import io
import json
import os

import numpy as np
import pytest
import torch

from ance_b200 import _lib
from ance_b200.optim import AdamW
from oracle.adamw_oracle import EagerAdamW, adamw_step_bounds, adamw_step_fp64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("kw,msg", [(dict(lr=-1e-3), "learning rate"), (dict(eps=-1.0), "epsilon"),
                                    (dict(betas=(1.0, 0.999)), "beta parameter: 1.0"),
                                    (dict(betas=(0.9, -0.1)), "beta parameter: -0.1")])
def test_hyperparameter_errors(kw, msg):
    p = torch.nn.Parameter(torch.zeros(3))
    for cls in (AdamW, EagerAdamW):
        with pytest.raises(ValueError, match=msg):
            cls([p], **kw)


def test_defaults_are_the_reference_class():
    for cls in (AdamW, EagerAdamW):
        opt = cls([torch.nn.Parameter(torch.zeros(3))])
        assert opt.defaults == dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True)
        assert opt.param_groups[0]["correct_bias"] is True
    opt = AdamW([{"params": [torch.nn.Parameter(torch.zeros(3))], "correct_bias": False}])
    assert opt.param_groups[0]["correct_bias"] is False


def test_cpu_parameters_are_refused_without_touching_the_gpu():
    p = torch.nn.Parameter(torch.ones(4))
    p.grad = torch.ones(4)
    opt = AdamW([p])
    with pytest.raises(_lib.AnceError, match="AdamW: .*no CPU fallback"):
        opt.step()
    q = torch.nn.Parameter(torch.ones(4))   # a parameter without a gradient is skipped, as in the reference
    opt = AdamW([q])
    assert opt.step(closure=lambda: 3.0) == 3.0 and len(opt.state[q]) == 0


def test_c_entry_point_argument_errors(lib):
    """Rejected before anything is enqueued, so no GPU is needed."""
    one = (C.c_void_p * 1)(0x1000)
    numel = (C.c_int64 * 1)(4)
    hyper = (C.c_double * 5)(1e-3, 0.9, 0.999, 1e-6, 0.0)
    assert lib.ance_adamw_step(0, None, None, None, None, None, None, None) == 0
    assert lib.ance_adamw_step(-1, one, one, one, one, numel, hyper, None) == 1
    assert b"< 0" in lib.ance_last_error()
    for k in range(6):   # each of the six arrays null
        args = [one, one, one, one, numel, hyper]
        args[k] = None
        assert lib.ance_adamw_step(1, *args, None) == 1
        assert b"null table array" in lib.ance_last_error()
    null = (C.c_void_p * 1)(0)
    assert lib.ance_adamw_step(1, one, null, one, one, numel, hyper, None) == 1
    assert b"null pointer" in lib.ance_last_error()
    assert lib.ance_adamw_step(1, one, null, null, null, (C.c_int64 * 1)(0), hyper, None) == 0   # numel 0: nothing to do
    bad = (C.c_int64 * 1)(-5)
    assert lib.ance_adamw_step(1, one, one, one, one, bad, hyper, None) == 1
    assert b"numel -5 < 0" in lib.ance_last_error()
    odd = (C.c_void_p * 1)(0x1002)
    for k in range(4):   # each of p, g, m, v misaligned
        args = [one, one, one, one]
        args[k] = odd
        assert lib.ance_adamw_step(1, *args, numel, hyper, None) == 1
        assert b"4-byte" in lib.ance_last_error()
    n = 513
    many = (C.c_void_p * n)(*([0x1000] * n))
    assert lib.ance_adamw_step(n, many, many, many, many, (C.c_int64 * n)(*([4] * n)), (C.c_double * (5 * n))(),
                               None) == _lib.ANCE_ERR_UNSUPPORTED
    assert b"at most 512" in lib.ance_last_error()
    hyp = (C.c_double * (5 * 17))(*[x for i in range(17) for x in (1e-3, 0.9, 0.999, 1e-6 * (i + 1), 0.0)])
    assert lib.ance_adamw_step(17, many, many, many, many, (C.c_int64 * 17)(*([4] * 17)), hyp,
                               None) == _lib.ANCE_ERR_UNSUPPORTED
    assert b"distinct (betas, eps)" in lib.ance_last_error()


@pytest.mark.parametrize("correct_bias", [True, False])
@pytest.mark.parametrize("weight_decay", [0.0, 0.01, -0.01])
def test_eager_oracle_agrees_with_fp64_to_fp32_rounding(correct_bias, weight_decay):
    """Ten eager fp32 steps, each replayed in fp64 from the eager state before it: p, m and v within adamw_step_bounds.
    A negative weight decay is no decay at all, as in the reference."""
    gen = torch.Generator().manual_seed(7)
    shapes = [(1,), (33,), (17, 9), (1001,)]
    params = [torch.nn.Parameter(torch.randn(s, generator=gen) * 0.5) for s in shapes]
    hp = dict(lr=3e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=weight_decay, correct_bias=correct_bias)
    opt = EagerAdamW(params, **hp)
    for step in range(1, 11):
        before = []
        for p in params:
            p.grad = torch.randn(p.shape, generator=gen) * 1e-2
            st = opt.state[p]
            before.append((p.detach().clone(), p.grad.clone(), st["exp_avg"].clone() if st else torch.zeros_like(p),
                           st["exp_avg_sq"].clone() if st else torch.zeros_like(p)))
        opt.step()
        for p, (p0, g, m0, v0) in zip(params, before):
            args = (hp["lr"], *hp["betas"], hp["eps"], weight_decay, correct_bias)
            out = adamw_step_fp64(p0, g, m0, v0, step, *args)
            tol_p, tol_m, tol_v = adamw_step_bounds(p0, g, m0, v0, out, step, *args)
            st = opt.state[p]
            assert st["step"] == step and isinstance(st["step"], int)
            assert (st["exp_avg"].double() - out[1]).abs().le(tol_m).all(), (p.shape, step)
            assert (st["exp_avg_sq"].double() - out[2]).abs().le(tol_v).all(), (p.shape, step)
            assert (p.detach().double() - out[0]).abs().le(tol_p).all(), (p.shape, step)


@pytest.fixture(scope="module")
def gold():
    z = np.load(os.path.join(ROOT, "tests", "golden", "lamb_steps.npz"))
    return {k: z[k] for k in z.files}, json.loads(str(z["meta"]))


def golden_group0(data, meta, cls, device="cpu"):
    """Group 0 of the golden Lamb run (lr 1e-2, eps 1e-8, no weight decay) as an AdamW without bias correction: the
    reference's Lamb with adam=True takes p <- p - lr m / (sqrt(v) + eps), which is that step."""
    params = {k: torch.nn.Parameter(torch.from_numpy(data[f"{k}/p0"]).to(device, copy=True))
              for k, s in meta["spec"].items() if s[1] == 0}
    g0 = meta["groups"][0]
    return params, cls(list(params.values()), lr=g0["lr"], eps=g0["eps"], correct_bias=False)


def golden_grads(params, data, s, device="cpu"):
    for k, p in params.items():
        g = data.get(f"{k}/g")
        p.grad = None if g is None else torch.from_numpy(g[s]).to(device, copy=True)


def within_trajectory_bound(p, ref, p0):
    """max |p - p_ref| <= 1e-4 max |p_ref - p0| (exact when the reference did not move the tensor)."""
    return float((p - ref).abs().max()) <= 1e-4 * float((ref - p0).abs().max())


def test_eager_oracle_follows_the_reference_adam_trajectory(gold):
    data, meta = gold
    assert meta["groups"][0] == {"lr": 1e-2, "eps": 1e-8}
    params, opt = golden_group0(data, meta, EagerAdamW)
    assert sorted(params) == ["bias_zero", "big_matrix", "no_grad", "zero_grad"]
    for s in range(meta["steps"]):
        golden_grads(params, data, s)
        opt.step()
        for k, p in params.items():
            p0 = torch.from_numpy(data[f"{k}/p0"])
            if f"{k}/g" not in data:
                assert torch.equal(p.detach(), p0) and len(opt.state[p]) == 0
                continue
            assert opt.state[p]["step"] == s + 1
            assert within_trajectory_bound(p.detach(), torch.from_numpy(data[f"adam/{k}/p"][s]), p0), (k, s)


def _reference_layout_state(params):
    """A state dict as the reference's AdamW writes it: int step, exp_avg, exp_avg_sq; correct_bias in the groups."""
    gen = torch.Generator().manual_seed(3)
    state = {i: {"step": 4 + i, "exp_avg": torch.randn(p.shape, generator=gen) * 1e-3,
                 "exp_avg_sq": torch.rand(p.shape, generator=gen) * 1e-6} for i, p in enumerate(params)}
    groups = [{"lr": 2e-5, "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": 0.01, "correct_bias": True,
               "params": list(range(len(params)))}]
    return {"state": state, "param_groups": groups}


def test_reference_layout_state_dicts_load():
    params = [torch.nn.Parameter(torch.zeros(s)) for s in ((5,), (3, 4))]
    sd = _reference_layout_state(params)
    buf = io.BytesIO()
    torch.save(sd, buf)
    for loaded in (sd, torch.load(io.BytesIO(buf.getvalue()))):
        for cls in (AdamW, EagerAdamW):
            opt = cls(params)
            opt.load_state_dict(loaded)
            g = opt.param_groups[0]
            assert (g["lr"], g["eps"], g["weight_decay"], g["correct_bias"]) == (2e-5, 1e-8, 0.01, True)
            for i, p in enumerate(params):
                st = opt.state[p]
                assert set(st) == {"step", "exp_avg", "exp_avg_sq"}
                assert st["step"] == 4 + i and type(st["step"]) is int
                assert torch.equal(st["exp_avg"], sd["state"][i]["exp_avg"])
                assert torch.equal(st["exp_avg_sq"], sd["state"][i]["exp_avg_sq"])
    # and what EagerAdamW saves, AdamW loads as it is
    opt = EagerAdamW(params, lr=1e-3)
    for p in params:
        p.grad = torch.ones_like(p)
    opt.step()
    buf = io.BytesIO()
    torch.save(opt.state_dict(), buf)
    ours = AdamW(params)
    ours.load_state_dict(torch.load(io.BytesIO(buf.getvalue())))
    for p in params:
        assert ours.state[p]["step"] == 1 and torch.equal(ours.state[p]["exp_avg"], opt.state[p]["exp_avg"])
    assert ours.param_groups[0]["lr"] == 1e-3
