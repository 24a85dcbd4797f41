"""ance_b200.optim.Lamb on the GPU: one step against the fp64 restatement (oracle/lamb_oracle.py) over the edge cases,
the reference's own 20-step trajectories (tests/golden/lamb_steps.npz), a RoBERTa-base-sized parameter set, bitwise
determinism, state-dict interop with the eager oracle in both directions, the absence of host synchronisations and of
torch kernels in a steady-state step, and 20 training steps of a small rdot_nll model."""
import io
import json
import os

import numpy as np
import pytest
import torch

from ance_b200.models import RobertaDot_NLL_LN
from ance_b200.optim import Lamb
from ance_b200.synthetic import random_roberta_state_dict, roberta_base_config
from oracle.lamb_oracle import EagerLamb, lamb_step_bounds, lamb_step_fp64

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"


def _view(n, offset, seed, std=0.02):
    """n elements that are a view at `offset` elements into a larger buffer (not 16-byte aligned for offset % 4 != 0)."""
    g = torch.Generator().manual_seed(seed)
    buf = (torch.randn(n + offset + 3, generator=g) * std).to(DEV)
    return buf[offset:offset + n]


def _param_view(n, offset, seed, std=0.02):
    return torch.nn.Parameter(_view(n, offset, seed, std))


def _rand(shape, seed, std):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * std).to(DEV)


def _check_step(opt, items, adam=False):
    """items: (param, group, p0, g, m0, v0) before opt.step() was called; checks the stepped state against fp64."""
    for p, grp, p0, g, m0, v0 in items:
        hp = (grp["lr"], *grp["betas"], grp["eps"], grp["weight_decay"])
        out = lamb_step_fp64(p0, g, m0, v0, *hp, adam=adam)
        tol_p, tol_m, tol_v = lamb_step_bounds(p0, g, m0, v0, out, *hp, adam=adam)
        p1, m1, v1, w, a, r = out
        st = opt.state[p]
        assert (st["exp_avg"].double() - m1).abs().le(tol_m).all(), p.shape
        assert (st["exp_avg_sq"].double() - v1).abs().le(tol_v).all(), p.shape
        assert (p.detach().double() - p1).abs().le(tol_p).all(), p.shape
        ws, As, rs = (float(st[k]) for k in ("weight_norm", "adam_norm", "trust_ratio"))
        assert abs(ws - w) <= 1e-6 * w and abs(As - a) <= 1e-6 * a, (p.shape, ws, w, As, a)
        assert abs(rs - r) <= 1e-6 * r, (p.shape, rs, r)
        assert all(st[k].dim() == 0 and st[k].is_cuda for k in ("weight_norm", "adam_norm", "trust_ratio"))


def _snapshot(opt, p):
    st = opt.state[p]
    if st:
        return p.detach().clone(), p.grad.clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone()
    return p.detach().clone(), p.grad.clone(), torch.zeros_like(p), torch.zeros_like(p)


@pytest.mark.parametrize("adam", [False, True])
def test_one_step_against_fp64_over_the_edge_cases(adam):
    big = 3 * 16384 + 5   # several blocks per tensor
    named = {
        "bias_zero": torch.nn.Parameter(torch.zeros(768, device=DEV)),                      # w = 0
        "clamped": torch.nn.Parameter(_rand((64, 96), 1, 1.0)),                             # ||p|| > 10
        "zero_grad": torch.nn.Parameter(_rand((33,), 2, 0.02)),                             # a = 0
        "no_grad": torch.nn.Parameter(_rand((7,), 3, 0.02)),                                # .grad None
        "one": torch.nn.Parameter(_rand((1,), 4, 0.5)),
        "empty": torch.nn.Parameter(torch.zeros(0, device=DEV)),
        "odd": torch.nn.Parameter(_rand((1001,), 5, 0.02)),
        "view_mixed": _param_view(big, 1, 6),         # p misaligned, its gradient and state aligned: scalar path
        "view_shared": _param_view(big, 3, 7),        # all four arrays at the same misalignment: head / body / tail
        "view_short": _param_view(2, 1, 8),            # shorter than its head
        "matrix_wd": torch.nn.Parameter(_rand((37, 53), 9, 0.5)),
    }
    groups = [{"params": [named[k] for k in ("bias_zero", "clamped", "zero_grad", "no_grad", "one", "empty",
                                            "view_short")], "lr": 2e-2, "eps": 1e-8},
              {"params": [named[k] for k in ("odd", "view_mixed", "view_shared", "matrix_wd")], "lr": 5e-2,
               "weight_decay": 1e-2}]
    opt = Lamb(groups, adam=adam)
    for i, (k, p) in enumerate(named.items()):
        if k != "no_grad":
            p.grad = torch.zeros_like(p) if k == "zero_grad" else _rand(p.shape, 100 + i, 1e-2)
    named["view_shared"].grad = _view(big, 3, 200, 1e-2)
    for k in ("exp_avg", "exp_avg_sq"):   # state at the same misalignment, from one earlier step's worth of moments
        opt.state[named["view_shared"]][k] = _view(big, 3, 300 + len(k), 1e-3).abs_()
    vs = named["view_shared"]
    assert {t.data_ptr() % 16 for t in (vs, vs.grad, opt.state[vs]["exp_avg"], opt.state[vs]["exp_avg_sq"])} == {12}
    opt.state[named["view_shared"]]["step"] = 1
    before = {k: _snapshot(opt, p) for k, p in named.items() if p.grad is not None}
    opt.step()
    torch.cuda.synchronize()
    gmap = {id(p): g for g in opt.param_groups for p in g["params"]}
    _check_step(opt, [(named[k], gmap[id(named[k])], *v) for k, v in before.items()], adam)
    assert len(opt.state[named["no_grad"]]) == 0
    st = opt.state
    assert float(st[named["bias_zero"]]["weight_norm"]) == 0 and float(st[named["bias_zero"]]["trust_ratio"]) == 1
    assert float(st[named["clamped"]]["weight_norm"]) == 10
    assert float(st[named["zero_grad"]]["adam_norm"]) == 0 and torch.equal(named["zero_grad"].detach(),
                                                                           before["zero_grad"][0])
    assert st[named["view_shared"]]["step"] == 2 and st[named["odd"]]["step"] == 1


@pytest.fixture(scope="module")
def gold():
    z = np.load(os.path.join(ROOT, "tests", "golden", "lamb_steps.npz"))
    return {k: z[k] for k in z.files}, json.loads(str(z["meta"]))


def _golden_setup(data, meta, cls, adam):
    params = {k: torch.nn.Parameter(torch.from_numpy(data[f"{k}/p0"]).to(DEV)) for k in meta["spec"]}
    groups = [dict(g, params=[params[k] for k, s in meta["spec"].items() if s[1] == gi])
              for gi, g in enumerate(meta["groups"])]
    return params, cls(groups, adam=adam)


def _golden_grads(params, data, s):
    for k, p in params.items():
        g = data.get(f"{k}/g")
        p.grad = None if g is None else torch.from_numpy(g[s]).to(DEV)


def _within_trajectory_bound(p, ref, p0):
    """max |p - p_ref| <= 1e-4 max |p_ref - p0| (exact when the reference did not move the tensor)."""
    return float((p - ref).abs().max()) <= 1e-4 * float((ref - p0).abs().max())


@pytest.mark.parametrize("run", ["lamb", "adam"])
def test_reference_trajectory(gold, run):
    data, meta = gold
    params, opt = _golden_setup(data, meta, Lamb, run == "adam")
    for s in range(meta["steps"]):
        _golden_grads(params, data, s)
        opt.step()
        for k, p in params.items():
            p0 = torch.from_numpy(data[f"{k}/p0"]).to(DEV)
            if f"{k}/g" not in data:
                assert torch.equal(p.detach(), p0) and len(opt.state[p]) == 0
                continue
            ref = torch.from_numpy(data[f"{run}/{k}/p"][s]).to(DEV)
            assert _within_trajectory_bound(p.detach(), ref, p0), (k, s)
            war = torch.tensor([float(opt.state[p][x]) for x in ("weight_norm", "adam_norm", "trust_ratio")])
            assert torch.allclose(war, torch.from_numpy(data[f"{run}/{k}/war"][s]), rtol=1e-5, atol=0), (k, s)


def _roberta_shapes():
    with torch.device("meta"):
        return [p.shape for p in RobertaDot_NLL_LN(roberta_base_config()).parameters()]


def test_roberta_base_sized_set_and_determinism():
    shapes = _roberta_shapes()
    assert len(shapes) == 201 and max(s.numel() for s in shapes) == 38_603_520
    params = [torch.nn.Parameter(_rand(s, i, 0.02 if len(s) == 2 else 0.5)) for i, s in enumerate(shapes)]
    opt = Lamb([{"params": params[::2], "lr": 1e-2, "eps": 1e-8},
                {"params": params[1::2], "lr": 3e-2, "eps": 1e-8, "weight_decay": 0.01}])
    for i, p in enumerate(params):
        p.grad = _rand(p.shape, 1000 + i, 1e-3)
    opt.step()                                     # moments from zero state, then the checked step from non-zero ones
    for i, p in enumerate(params):
        p.grad = _rand(p.shape, 2000 + i, 1e-3)
    before = [_snapshot(opt, p) for p in params]
    opt.step()
    torch.cuda.synchronize()
    gmap = {id(p): g for g in opt.param_groups for p in g["params"]}
    _check_step(opt, [(p, gmap[id(p)], *b) for p, b in zip(params, before)])
    # bitwise determinism: the same step again from the same state
    after = [(p.detach().clone(), opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone()) for p in params]
    norms = opt._norms.clone()
    for p, (p0, _, m0, v0) in zip(params, before):
        p.data.copy_(p0)
        opt.state[p]["exp_avg"].copy_(m0)
        opt.state[p]["exp_avg_sq"].copy_(v0)
    opt.step()
    torch.cuda.synchronize()
    for p, (p1, m1, v1) in zip(params, after):
        assert torch.equal(p.detach(), p1) and torch.equal(opt.state[p]["exp_avg"], m1)
        assert torch.equal(opt.state[p]["exp_avg_sq"], v1)
    assert torch.equal(opt._norms, norms)


@pytest.mark.parametrize("first,second", [(EagerLamb, Lamb), (Lamb, EagerLamb)])
def test_state_dict_interop(gold, first, second):
    data, meta = gold
    params, opt = _golden_setup(data, meta, first, False)
    for s in range(3):
        _golden_grads(params, data, s)
        opt.step()
    buf = io.BytesIO()
    torch.save(opt.state_dict(), buf)
    opt2 = second([{"params": g["params"]} for g in opt.param_groups])
    opt2.load_state_dict(torch.load(io.BytesIO(buf.getvalue())))
    for s in range(3, 6):
        _golden_grads(params, data, s)
        opt2.step()
    for cls in (EagerLamb, Lamb):   # six steps of either alone
        ref_params, ref = _golden_setup(data, meta, cls, False)
        for s in range(6):
            _golden_grads(ref_params, data, s)
            ref.step()
        for k, p in params.items():
            p0 = torch.from_numpy(data[f"{k}/p0"]).to(DEV)
            assert _within_trajectory_bound(p.detach(), ref_params[k].detach(), p0), (cls.__name__, k)
            if f"{k}/g" in data:
                assert opt2.state[p]["step"] == 6


def _set(n, seed):
    params = [torch.nn.Parameter(_rand((257 + 31 * i,), seed + i, 0.02)) for i in range(n)]
    opt = Lamb(params, lr=1e-3, eps=1e-8)
    for i, p in enumerate(params):
        p.grad = _rand(p.shape, seed + 500 + i, 1e-3)
    opt.step()   # state allocated: the following steps are steady-state
    torch.cuda.synchronize()
    return opt


def test_steady_state_step_does_not_synchronise():
    opt = _set(300, 0)
    ev = torch.cuda.Event()
    torch.cuda._sleep(200_000_000)   # ~100 ms of device time ahead of the step
    ev.record()
    opt.step()
    pending = not ev.query()
    torch.cuda.synchronize()
    assert pending, "step() waited for earlier work on the stream"
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            opt.step()
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()


def test_steady_state_step_launches_only_the_library_kernels():
    from torch.profiler import ProfilerActivity, profile
    counts = {}
    for n in (3, 300):
        opt = _set(n, 10 * n)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            opt.step()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        assert names and all("lamb_" in x for x in names), names
        counts[n] = len(names)
    assert counts[3] == counts[300] == 3, counts


def test_small_rdot_nll_trains_like_the_eager_oracle():
    cfg = roberta_base_config(num_hidden_layers=2, vocab_size=1000)
    sd = random_roberta_state_dict(seed=0, n_layer=2, vocab=1000)
    gen = torch.Generator().manual_seed(0)

    def batch(B, L):
        ids = torch.randint(3, 1000, (B, L), generator=gen)
        ids[:, 0] = 0
        return ids.to(DEV), torch.ones(B, L, dtype=torch.int64, device=DEV)

    q, a, b = batch(8, 32), batch(8, 64), batch(8, 64)
    losses = {}
    for cls in (Lamb, EagerLamb):
        m = RobertaDot_NLL_LN(cfg)
        m.load_state_dict(sd, strict=True)
        m = m.to(DEV)
        m.set_trainable(True)
        opt = cls(m.parameters(), lr=5e-3, eps=1e-8)
        losses[cls] = []
        for _ in range(20):
            m.zero_grad(set_to_none=True)
            (loss,) = m(q[0], q[1], a[0], a[1], b[0], b[1])
            loss.backward()
            opt.step()
            losses[cls].append(float(loss.detach()))
    ours, ref = np.array(losses[Lamb]), np.array(losses[EagerLamb])
    assert np.abs(ours - ref).max() <= 1e-3, (ours, ref)
    assert ours[-1] < ours[0] - 0.01, ours   # the encoder sees the weights the kernel wrote
