"""ance_b200.optim.AdamW on the GPU: one step against the fp64 restatement (oracle/adamw_oracle.py) over the edge cases
and hyperparameters, the reference's own adam trajectory (group 0 of tests/golden/lamb_steps.npz), a 20-step trajectory
of the eager restatement with bias correction and weight decay, a RoBERTa-base-sized set and one of more than 512
tensors, bitwise determinism, state-dict interop with the eager restatement in both directions, the absence of host
synchronisations and of torch kernels in a steady-state step, and 20 training steps of a small DPR BiEncoder."""
import io
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from ance_b200 import _lib
from ance_b200.models import BiEncoder, RobertaDot_NLL_LN
from ance_b200.optim import AdamW
from ance_b200.synthetic import random_roberta_state_dict, roberta_base_config
from oracle.adamw_oracle import EagerAdamW, adamw_step_bounds, adamw_step_fp64
from tests.test_adamw_cpu import golden_grads, golden_group0, gold, within_trajectory_bound  # noqa: F401

pytestmark = pytest.mark.gpu
DEV = "cuda"
LR = 1e-6   # small enough that 20 steps stay on the smooth part of the loss


def _view(n, offset, seed, std=0.02):
    """n elements that are a view at `offset` elements into a larger buffer (not 16-byte aligned for offset % 4 != 0)."""
    g = torch.Generator().manual_seed(seed)
    buf = (torch.randn(n + offset + 3, generator=g) * std).to(DEV)
    return buf[offset:offset + n]


def _rand(shape, seed, std):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * std).to(DEV)


def _snapshot(opt, p):
    st = opt.state[p]
    if st:
        return p.detach().clone(), p.grad.clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone()
    return p.detach().clone(), p.grad.clone(), torch.zeros_like(p), torch.zeros_like(p)


def _check_step(opt, items):
    """items: (param, group, p0, g, m0, v0) before opt.step() was called; checks the stepped state against fp64."""
    for p, grp, p0, g, m0, v0 in items:
        st = opt.state[p]
        hp = (st["step"], grp["lr"], *grp["betas"], grp["eps"], grp["weight_decay"], grp["correct_bias"])
        out = adamw_step_fp64(p0, g, m0, v0, *hp)
        tol_p, tol_m, tol_v = adamw_step_bounds(p0, g, m0, v0, out, *hp)
        assert (st["exp_avg"].double() - out[1]).abs().le(tol_m).all(), p.shape
        assert (st["exp_avg_sq"].double() - out[2]).abs().le(tol_v).all(), p.shape
        assert (p.detach().double() - out[0]).abs().le(tol_p).all(), (p.shape, hp)


def _step_and_check(opt, params):
    gmap = {id(p): g for g in opt.param_groups for p in g["params"]}
    before = [(p, _snapshot(opt, p)) for p in params if p.grad is not None]
    opt.step()
    torch.cuda.synchronize()
    _check_step(opt, [(p, gmap[id(p)], *b) for p, b in before])
    return before


@pytest.mark.parametrize("eps", [1e-6, 1e-8])
@pytest.mark.parametrize("weight_decay", [0.0, 0.01, -0.01])
@pytest.mark.parametrize("correct_bias", [True, False])
def test_one_step_against_fp64_over_the_edge_cases(correct_bias, weight_decay, eps):
    big = 3 * 16384 + 5   # several blocks per tensor
    named = {
        "zero": torch.nn.Parameter(torch.zeros(768, device=DEV)),
        "zero_grad": torch.nn.Parameter(_rand((33,), 2, 0.02)),
        "no_grad": torch.nn.Parameter(_rand((7,), 3, 0.02)),
        "one": torch.nn.Parameter(_rand((1,), 4, 0.5)),
        "empty": torch.nn.Parameter(torch.zeros(0, device=DEV)),
        "odd": torch.nn.Parameter(_rand((1001,), 5, 0.02)),
        "blocks": torch.nn.Parameter(_rand((big,), 6, 0.02)),
        "view_mixed": torch.nn.Parameter(_view(big, 1, 7)),    # p misaligned, its gradient and state aligned: scalar path
        "view_shared": torch.nn.Parameter(_view(big, 3, 8)),   # all four arrays at the same misalignment
        "view_short": torch.nn.Parameter(_view(2, 1, 9)),      # shorter than its head
        "matrix": torch.nn.Parameter(_rand((37, 53), 10, 0.5)),
    }
    groups = [{"params": [named[k] for k in ("zero", "zero_grad", "no_grad", "one", "empty", "view_short")],
               "lr": 2e-2},
              {"params": [named[k] for k in ("odd", "blocks", "view_mixed", "view_shared", "matrix")], "lr": 5e-2,
               "weight_decay": weight_decay}]
    opt = AdamW(groups, eps=eps, correct_bias=correct_bias)
    for i, (k, p) in enumerate(named.items()):
        if k != "no_grad":
            p.grad = torch.zeros_like(p) if k == "zero_grad" else _rand(p.shape, 100 + i, 1e-2)
    vs = named["view_shared"]
    vs.grad = _view(big, 3, 200, 1e-2)
    st = opt.state[vs]   # a preloaded state at step 5, at the same misalignment, next to fresh ones
    st["step"] = 5
    st["exp_avg"] = _view(big, 3, 301, 1e-3)
    st["exp_avg_sq"] = _view(big, 3, 302, 1e-3).square_()
    assert {t.data_ptr() % 16 for t in (vs, vs.grad, st["exp_avg"], st["exp_avg_sq"])} == {12}
    zg0 = named["zero_grad"].detach().clone()
    launches = _lib.load().ance_launch_count()
    _step_and_check(opt, list(named.values()))
    assert _lib.load().ance_launch_count() - launches == 1
    assert len(opt.state[named["no_grad"]]) == 0
    assert opt.state[vs]["step"] == 6 and opt.state[named["odd"]]["step"] == 1
    assert torch.equal(named["zero_grad"].detach(), zg0)   # zero state and gradient: the step leaves it as it was


@pytest.mark.parametrize("correct_bias", [True, False])
def test_steps_bit_identical_to_the_eager_step(correct_bias):
    """The kernel rounds each operation as torch's CUDA kernels round the eager step (csrc/optim.cu, adamw_update), so
    three steps over 4M+ elements, decayed and not, aligned and not, give the eager step's p, m and v bit for bit."""
    shapes = [(1 << 22,), (1001,), (768, 3072), (64,)]
    ours = [torch.nn.Parameter(_rand(s, i, 0.05)) for i, s in enumerate(shapes)] + [torch.nn.Parameter(_view(5003, 1, 9))]
    ref = [torch.nn.Parameter(p.detach().clone()) for p in ours]

    def groups(ps):
        return [{"params": ps[:3], "lr": 1e-3, "weight_decay": 0.01}, {"params": ps[3:], "lr": 3e-5}]

    opt, eager = AdamW(groups(ours), eps=1e-8, correct_bias=correct_bias), EagerAdamW(groups(ref), eps=1e-8,
                                                                                     correct_bias=correct_bias)
    for s in range(3):
        for i, (p, r) in enumerate(zip(ours, ref)):
            p.grad = _rand(p.shape, 100 * s + i, 1e-3 * (i + 1))
            r.grad = p.grad.clone()
        opt.step()
        eager.step()
        for p, r in zip(ours, ref):
            assert torch.equal(p.detach(), r.detach()), (p.shape, s)
            assert torch.equal(opt.state[p]["exp_avg"], eager.state[r]["exp_avg"]), (p.shape, s)
            assert torch.equal(opt.state[p]["exp_avg_sq"], eager.state[r]["exp_avg_sq"]), (p.shape, s)


def test_more_than_16_groups_in_one_call():
    """20 groups of their own lr and weight decay and mixed step counts: one launch, each tensor against fp64."""
    params = [torch.nn.Parameter(_rand((513 + 7 * i,), i, 0.05)) for i in range(20)]
    opt = AdamW([{"params": [p], "lr": 1e-3 * (i + 1), "weight_decay": 0.01 * (i % 3)} for i, p in enumerate(params)],
                eps=1e-8)
    for i, p in enumerate(params):
        p.grad = _rand(p.shape, 100 + i, 1e-3)
        if i % 2:
            st = opt.state[p]
            st["step"], st["exp_avg"], st["exp_avg_sq"] = i, _rand(p.shape, 200 + i, 1e-4), _rand(p.shape, 300 + i,
                                                                                                  1e-4).square()
    launches = _lib.load().ance_launch_count()
    _step_and_check(opt, params)
    assert _lib.load().ance_launch_count() - launches == 1
    assert [opt.state[p]["step"] for p in params] == [i + 1 if i % 2 else 1 for i in range(20)]


def test_reference_trajectory(gold):
    data, meta = gold
    params, opt = golden_group0(data, meta, AdamW, DEV)
    for s in range(meta["steps"]):
        golden_grads(params, data, s, DEV)
        opt.step()
        for k, p in params.items():
            p0 = torch.from_numpy(data[f"{k}/p0"]).to(DEV)
            if f"{k}/g" not in data:
                assert torch.equal(p.detach(), p0) and len(opt.state[p]) == 0
                continue
            assert opt.state[p]["step"] == s + 1
            ref = torch.from_numpy(data[f"adam/{k}/p"][s]).to(DEV)
            assert within_trajectory_bound(p.detach(), ref, p0), (k, s)


def _pair(seed, n=6):
    shapes = [(768,), (64, 96), (1001,), (3, 16384 + 3), (1,), (2, 5)]
    return [[torch.nn.Parameter(_rand(s, seed + i, 0.05)) for i, s in enumerate(shapes[:n])] for _ in range(2)]


def _groups(params):
    return [{"params": [p for p in params if p.dim() > 1], "weight_decay": 0.01},
            {"params": [p for p in params if p.dim() <= 1], "weight_decay": 0.0}]


def _grads(params, s):
    for i, p in enumerate(params):
        p.grad = _rand(p.shape, 1000 * s + i, 1e-3 * (1 + i))


def test_eager_trajectory_with_bias_correction_and_weight_decay():
    ours_p, ref_p = _pair(0)
    p0 = [p.detach().clone() for p in ours_p]
    ours, ref = AdamW(_groups(ours_p), lr=3e-3), EagerAdamW(_groups(ref_p), lr=3e-3)
    for s in range(20):
        _grads(ours_p, s)
        _grads(ref_p, s)
        ours.step()
        ref.step()
        for a, b, z in zip(ours_p, ref_p, p0):
            assert within_trajectory_bound(a.detach(), b.detach(), z), (a.shape, s)
            assert ours.state[a]["step"] == ref.state[b]["step"] == s + 1


def _roberta_shapes():
    with torch.device("meta"):
        return [p.shape for p in RobertaDot_NLL_LN(roberta_base_config()).parameters()]


def test_roberta_base_sized_set_and_determinism():
    shapes = _roberta_shapes()
    assert len(shapes) == 201 and max(s.numel() for s in shapes) == 38_603_520
    params = [torch.nn.Parameter(_rand(s, i, 0.02 if len(s) == 2 else 0.5)) for i, s in enumerate(shapes)]
    opt = AdamW([{"params": params[::2], "lr": 1e-2, "eps": 1e-8},
                 {"params": params[1::2], "lr": 3e-2, "eps": 1e-8, "weight_decay": 0.01}])
    for i, p in enumerate(params):
        p.grad = _rand(p.shape, 1000 + i, 1e-3)
    opt.step()                                     # moments from zero state, then the checked step from non-zero ones
    for i, p in enumerate(params):
        p.grad = _rand(p.shape, 2000 + i, 1e-3)
    before = [b for _, b in _step_and_check(opt, params)]
    # bitwise determinism: the same step again from the same state
    after = [(p.detach().clone(), opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone()) for p in params]
    for p, (p0, _, m0, v0) in zip(params, before):
        p.data.copy_(p0)
        opt.state[p]["exp_avg"].copy_(m0)
        opt.state[p]["exp_avg_sq"].copy_(v0)
        opt.state[p]["step"] -= 1
    opt.step()
    torch.cuda.synchronize()
    for p, (p1, m1, v1) in zip(params, after):
        assert torch.equal(p.detach(), p1) and torch.equal(opt.state[p]["exp_avg"], m1)
        assert torch.equal(opt.state[p]["exp_avg_sq"], v1)


def test_more_than_512_tensors_split_the_call():
    params = [torch.nn.Parameter(_rand((97 + (i % 13),), i, 0.05)) for i in range(600)]
    opt = AdamW(_groups(params), lr=1e-3)
    for i, p in enumerate(params):
        p.grad = _rand(p.shape, 5000 + i, 1e-3)
    opt.step()
    for i, p in enumerate(params):
        p.grad = _rand(p.shape, 7000 + i, 1e-3)
    launches = _lib.load().ance_launch_count()
    _step_and_check(opt, params)
    assert _lib.load().ance_launch_count() - launches == 2


@pytest.mark.parametrize("first,second", [(EagerAdamW, AdamW), (AdamW, EagerAdamW)])
def test_state_dict_interop(first, second):
    params, ref_params = _pair(50)
    opt = first(_groups(params), lr=3e-3)
    for s in range(3):
        _grads(params, s)
        opt.step()
    buf = io.BytesIO()
    torch.save(opt.state_dict(), buf)
    opt2 = second([{"params": g["params"]} for g in opt.param_groups])
    opt2.load_state_dict(torch.load(io.BytesIO(buf.getvalue())))
    assert all(type(opt2.state[p]["step"]) is int for p in params)
    for s in range(3, 6):
        _grads(params, s)
        opt2.step()
    p0 = [p.detach().clone() for p in ref_params]
    for cls in (EagerAdamW, AdamW):   # six steps of either alone
        ref_ps = [torch.nn.Parameter(p.clone()) for p in p0]
        ref = cls(_groups(ref_ps), lr=3e-3)
        for s in range(6):
            _grads(ref_ps, s)
            ref.step()
        for p, r, z in zip(params, ref_ps, p0):
            assert within_trajectory_bound(p.detach(), r.detach(), z), (cls.__name__, p.shape)
            assert opt2.state[p]["step"] == 6


def _set(n, seed):
    params = [torch.nn.Parameter(_rand((257 + 31 * i,), seed + i, 0.02)) for i in range(n)]
    opt = AdamW(_groups(params), lr=1e-3, eps=1e-8)
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


def _kernel_names():
    """Child-process half of test_steady_state_step_launches_only_the_library_kernel: one steady-state step of 3 and of
    300 tensors under torch.profiler; prints one JSON line {n: [GPU activity names]}."""
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for n in (3, 300):
        opt = _set(n, 10 * n)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            opt.step()
            torch.cuda.synchronize()
        out[n] = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    print(json.dumps(out))


def test_steady_state_step_launches_only_the_library_kernel():
    """One `adamw_` kernel per call and nothing else, at 3 and at 300 tensors.  The names come from torch.profiler in a
    child process, as in test_gpu_gemm_wide.py, so that this test leaves no profiler state behind: a later session in the
    same process (test_gpu_lamb.py reads kernel names too) has been seen to miss GPU activity after earlier ones."""
    root = Path(__file__).resolve().parent.parent
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(root)] + [os.environ.get("PYTHONPATH", "")]))
    r = subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c",
                        "from tests.test_gpu_adamw import _kernel_names; _kernel_names()"],
                       cwd=root, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    for n in ("3", "300"):
        assert len(names[n]) == 1 and "adamw_" in names[n][0], names


def test_small_dpr_biencoder_trains_like_the_eager_oracle():
    """20 in-batch training steps of a 2-layer DPR BiEncoder (8 pairs at up to 256 tokens) with dpr_utils.get_optimizer's
    two groups (weight decay 0.01 except on biases and LayerNorm weights) and clipping at 1.  One copy of the model takes
    the fused step and a second copy the eager one, both from the first copy's clipped gradients, so the two trajectories
    differ by the optimizers alone: the encoder's word / position gradients are scatter-added with fp32 atomics, and Adam
    would turn their run-to-run last-bit differences into diverging trajectories of two independent runs."""
    vocab = 1000
    sd = {**random_roberta_state_dict(seed=11, n_layer=2, vocab=vocab, max_pos=512, head=False,
                                      prefix="question_model."),
          **random_roberta_state_dict(seed=12, n_layer=2, vocab=vocab, max_pos=512, head=False, prefix="ctx_model.")}
    gen = torch.Generator().manual_seed(0)

    def batch(B, L):
        lens = torch.randint(L // 2, L + 1, (B,), generator=gen)
        mask = torch.arange(L)[None, :] < lens[:, None]
        ids = torch.where(mask, torch.randint(3, vocab, (B, L), generator=gen), torch.zeros(B, L, dtype=torch.int64))
        ids[:, 0] = 101
        return ids.to(DEV), mask.long().to(DEV)

    q, a = batch(8, 256), batch(8, 256)
    models, opts = [], []
    for cls in (AdamW, EagerAdamW):
        m = BiEncoder(type("A", (), {"num_hidden_layers": 2, "vocab_size": vocab})())
        m.load_state_dict(sd)
        m = m.to(DEV)
        m.set_trainable(True, max_len=256)
        no_decay = ("bias", "LayerNorm.weight")
        opts.append(cls([{"params": [p for n, p in m.named_parameters() if not any(k in n for k in no_decay)],
                          "weight_decay": 0.01},
                         {"params": [p for n, p in m.named_parameters() if any(k in n for k in no_decay)],
                          "weight_decay": 0.0}], lr=LR))
        models.append(m)

    def loss_of(m):
        eq, ea = m(q[0], q[1], a[0], a[1])
        return -torch.log_softmax(eq @ ea.T, dim=1).diagonal().mean()

    losses = {"fused": [], "eager": []}
    for _ in range(20):
        models[0].zero_grad(set_to_none=True)
        loss = loss_of(models[0])
        loss.backward()
        torch.nn.utils.clip_grad_norm_(models[0].parameters(), 1.0)
        # a training forward, which reads the parameters' current values: the eager step writes through p.data and bumps
        # no version counter, so the inference path's cached weights would not see it
        losses["eager"].append(float(loss_of(models[1]).detach()))
        for p, r in zip(models[0].parameters(), models[1].parameters()):
            r.grad = None if p.grad is None else p.grad.clone()
        for opt in opts:
            opt.step()
        losses["fused"].append(float(loss.detach()))
    ours, ref = np.array(losses["fused"]), np.array(losses["eager"])
    assert np.abs(ours - ref).max() <= 1e-3, (ours, ref)
    assert ours[-1] < ours[0] - 0.01, ours   # the encoder sees the weights the kernel wrote
