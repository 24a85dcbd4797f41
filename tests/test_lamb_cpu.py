"""Lamb without a GPU: the oracle's two restatements against the reference's own trajectory (tests/golden/lamb_steps.npz,
written by oracle/make_golden_lamb.py from utils/lamb.py), the constructor's checks, the refusals of CPU tensors and
the C entry point's argument errors."""
import ctypes as C
import io
import json
import os

import numpy as np
import pytest
import torch

from ance_b200 import _lib
from ance_b200.optim import Lamb, log_lamb_rs
from oracle.lamb_oracle import EagerLamb, lamb_step_bounds, lamb_step_fp64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold():
    z = np.load(os.path.join(ROOT, "tests", "golden", "lamb_steps.npz"))
    return {k: z[k] for k in z.files}, json.loads(str(z["meta"]))


def _setup(gold_data, meta, cls, adam):
    params = {k: torch.nn.Parameter(torch.from_numpy(gold_data[f"{k}/p0"]).clone()) for k in meta["spec"]}
    groups = [dict(g, params=[params[k] for k, s in meta["spec"].items() if s[1] == gi])
              for gi, g in enumerate(meta["groups"])]
    return params, cls(groups, adam=adam)


def _set_grads(params, gold_data, step):
    for k, p in params.items():
        g = gold_data.get(f"{k}/g")
        p.grad = None if g is None else torch.from_numpy(g[step]).clone()


@pytest.mark.parametrize("run", ["lamb", "adam"])
def test_eager_oracle_reproduces_the_reference_bit_for_bit(gold, run):
    data, meta = gold
    params, opt = _setup(data, meta, EagerLamb, run == "adam")
    for s in range(meta["steps"]):
        _set_grads(params, data, s)
        opt.step()
        for k, p in params.items():
            if f"{k}/g" not in data:
                assert len(opt.state[p]) == 0 and torch.equal(p.detach(), torch.from_numpy(data[f"{k}/p0"]))
                continue
            st = opt.state[p]
            assert st["step"] == s + 1
            assert np.array_equal(p.detach().numpy(), data[f"{run}/{k}/p"][s]), (k, s)
            assert np.array_equal(st["exp_avg"].numpy(), data[f"{run}/{k}/m"][s]), (k, s)
            assert np.array_equal(st["exp_avg_sq"].numpy(), data[f"{run}/{k}/v"][s]), (k, s)
            war = np.array([float(st[x]) for x in ("weight_norm", "adam_norm", "trust_ratio")], dtype=np.float32)
            assert np.array_equal(war, data[f"{run}/{k}/war"][s]), (k, s)


@pytest.mark.parametrize("run", ["lamb", "adam"])
def test_fp64_restatement_agrees_with_the_reference_to_fp32_rounding(gold, run):
    """Each golden step, replayed in fp64 from the golden state before it: m, v and p within lamb_step_bounds (2 ulp of
    the operands' scale, carried through u), w and a within 1e-6 relative, r within 2e-6.  The edge cases come out as the
    reference took them."""
    data, meta = gold
    seen = set()
    for k, (shape, gi, _, _) in meta["spec"].items():
        if f"{k}/g" not in data:
            continue
        grp = {**dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0), **meta["groups"][gi]}
        p, m, v = data[f"{k}/p0"], np.zeros(shape, np.float32), np.zeros(shape, np.float32)
        for s in range(meta["steps"]):
            g = data[f"{k}/g"][s]
            args = [torch.from_numpy(x) for x in (p, g, m, v)]
            hp = (grp["lr"], *grp["betas"], grp["eps"], grp["weight_decay"])
            out = lamb_step_fp64(*args, *hp, adam=run == "adam")
            tol_p, tol_m, tol_v = (x.numpy() for x in lamb_step_bounds(*args, out, *hp, adam=run == "adam"))
            p1, m1, v1, w, a, r = out
            ref = {f: data[f"{run}/{k}/{f}"][s] for f in ("p", "m", "v", "war")}
            assert (np.abs(m1.numpy() - ref["m"]) <= tol_m).all(), (k, s)
            assert (np.abs(v1.numpy() - ref["v"]) <= tol_v).all(), (k, s)
            assert abs(w - ref["war"][0]) <= 1e-6 * w and abs(a - ref["war"][1]) <= 1e-6 * a, (k, s)
            assert abs(r - ref["war"][2]) <= 2e-6 * r, (k, s)
            assert (np.abs(p1.numpy() - ref["p"]) <= tol_p).all(), (k, s)
            seen.update({"w0"} if w == 0 else set())
            seen.update({"clamp"} if w == 10.0 else set())
            seen.update({"a0"} if a == 0 else set())
            p, m, v = ref["p"], ref["m"], ref["v"]
    assert seen == {"w0", "clamp", "a0"}


@pytest.mark.parametrize("kw,msg", [(dict(lr=-1e-3), "learning rate"), (dict(eps=-1.0), "epsilon"),
                                    (dict(betas=(1.0, 0.999)), "index 0"), (dict(betas=(0.9, -0.1)), "index 1")])
def test_hyperparameter_errors(kw, msg):
    p = torch.nn.Parameter(torch.zeros(3))
    for cls in (Lamb, EagerLamb):
        with pytest.raises(ValueError, match=msg):
            cls([p], **kw)


def test_defaults_are_the_reference_class():
    opt = Lamb([torch.nn.Parameter(torch.zeros(3))])
    assert opt.defaults == dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0) and opt.adam is False


def test_cpu_parameters_are_refused_without_touching_the_gpu():
    p = torch.nn.Parameter(torch.ones(4))
    p.grad = torch.ones(4)
    opt = Lamb([p])
    with pytest.raises(_lib.AnceError, match="no CPU fallback"):
        opt.step()
    q = torch.nn.Parameter(torch.ones(4))   # a parameter without a gradient is skipped, as in the reference
    assert Lamb([q]).step(closure=lambda: 3.0) == 3.0


def test_state_dict_of_the_eager_oracle_loads(gold):
    data, meta = gold
    params, opt = _setup(data, meta, EagerLamb, False)
    for s in range(2):
        _set_grads(params, data, s)
        opt.step()
    buf = io.BytesIO()
    torch.save(opt.state_dict(), buf)
    ours = Lamb([dict(g) for g in opt.param_groups])
    ours.load_state_dict(torch.load(io.BytesIO(buf.getvalue())))
    for p in params.values():
        assert set(ours.state[p]) == set(opt.state[p])
        if opt.state[p]:
            assert ours.state[p]["step"] == 2 and torch.equal(ours.state[p]["exp_avg"], opt.state[p]["exp_avg"])


def test_log_lamb_rs_reads_the_state_keys(gold):
    data, meta = gold
    params, opt = _setup(data, meta, EagerLamb, False)
    _set_grads(params, data, 0)
    opt.step()
    got = {}

    class Writer:
        def add_histogram(self, tag, values, step):
            got[tag] = (values, step)

    log_lamb_rs(opt, Writer(), 123)
    assert sorted(got) == ["lamb/adam_norm", "lamb/trust_ratio", "lamb/weight_norm"]
    assert got["lamb/trust_ratio"][1] == 123 and got["lamb/weight_norm"][0].numel() == 6   # no_grad has no state


def test_c_entry_point_argument_errors(lib):
    """Rejected before anything is enqueued, so no GPU is needed."""
    one = (C.c_void_p * 1)(0x1000)
    numel = (C.c_int64 * 1)(4)
    hyper = (C.c_double * 5)(1e-3, 0.9, 0.999, 1e-6, 0.0)
    out = C.c_void_p(0x2000)
    assert lib.ance_lamb_step(0, None, None, None, None, None, None, 0, None, None) == 0
    assert lib.ance_lamb_step(-1, one, one, one, one, numel, hyper, 0, out, None) == 1
    assert b"< 0" in lib.ance_last_error()
    null = (C.c_void_p * 1)(0)
    assert lib.ance_lamb_step(1, one, null, one, one, numel, hyper, 0, out, None) == 1
    assert b"null pointer" in lib.ance_last_error()
    bad = (C.c_int64 * 1)(-5)
    assert lib.ance_lamb_step(1, one, one, one, one, bad, hyper, 0, out, None) == 1
    odd = (C.c_void_p * 1)(0x1002)
    assert lib.ance_lamb_step(1, odd, one, one, one, numel, hyper, 0, out, None) == 1
    assert b"4-byte" in lib.ance_last_error()
    assert lib.ance_lamb_step(1, one, one, one, one, numel, None, 0, out, None) == 1
    n = 513
    many = (C.c_void_p * n)(*([0x1000] * n))
    assert lib.ance_lamb_step(n, many, many, many, many, (C.c_int64 * n)(*([4] * n)), (C.c_double * (5 * n))(),
                              0, out, None) == _lib.ANCE_ERR_UNSUPPORTED
    assert b"at most 512" in lib.ance_last_error()
    hyp = (C.c_double * (5 * 17))(*[x for i in range(17) for x in (1e-3 * (i + 1), 0.9, 0.999, 1e-6, 0.0)])
    assert lib.ance_lamb_step(17, many, many, many, many, (C.c_int64 * 17)(*([4] * 17)), hyp, 0, out,
                              None) == _lib.ANCE_ERR_UNSUPPORTED
    assert b"distinct" in lib.ance_last_error()
