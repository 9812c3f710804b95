"""The optimizer replays of tests/optim_ref.py against torch.optim on the CPU (host only): the float64 formulas match torch.optim.SGD
and torch.optim.AdamW run in float64 over every option combination (first-step clone, dampening, nesterov, decoupled decay, bias
corrections, an lr that changes each step), and the float32 replay, the device's exact order of operations, stays within a few ulps of
torch's float32 CPU optimizers.  Also the ResNet-18 table used by the GPU tests and the benchmark."""
import itertools

import numpy as np
import pytest
import torch

import optim_ref as R

STEPS = 20
SHAPES = [(7,), (64, 3), (5, 4, 3)]


def grads(seed, dtype):
    rng = np.random.default_rng(seed)
    return [[rng.standard_normal(s).astype(dtype) for s in SHAPES] for _ in range(STEPS)]


def lrs(base):
    return [base * (1.0 + 0.5 * np.sin(i)) for i in range(STEPS)]


def torch_run(dtype, make, gs, lr_seq, seed):
    rng = np.random.default_rng(seed + 1)
    ps = [torch.from_numpy(rng.standard_normal(s).astype(dtype)).requires_grad_(True) for s in SHAPES]
    p0 = [p.detach().numpy().copy() for p in ps]
    opt = make(ps)
    for gstep, lr in zip(gs, lr_seq):
        opt.param_groups[0]["lr"] = lr
        for p, g in zip(ps, gstep):
            p.grad = torch.from_numpy(g.copy())
        opt.step()
    return p0, [p.detach().numpy() for p in ps], opt


SGD_CASES = [(mu, d, n, wd) for mu, d, n, wd in itertools.product((0.0, 0.9), (0.0, 0.1), (False, True), (0.0, 1e-2))
             if not n or (mu > 0 and d == 0)]
ADAM_CASES = [(b, wd, eps) for b, wd, eps in itertools.product(((0.9, 0.999), (0.8, 0.99)), (0.0, 1e-2), (1e-8, 1e-3))]


def replay_sgd(fn, p0, gs, lr_seq, mu, d, n, wd):
    out = []
    for p, k in zip(p0, range(len(SHAPES))):
        b = None
        for t, (gstep, lr) in enumerate(zip(gs, lr_seq), 1):
            p, b = fn(p, gstep[k], b, lr, t, mu, d, n, wd)
        out.append(p)
    return out


def replay_adamw(fn, p0, gs, lr_seq, betas, wd, eps, dtype):
    out = []
    for p, k in zip(p0, range(len(SHAPES))):
        m, v = np.zeros_like(p), np.zeros_like(p)
        for t, (gstep, lr) in enumerate(zip(gs, lr_seq), 1):
            p, m, v = fn(p, gstep[k], m, v, lr, t, betas[0], betas[1], eps, wd)
        out.append(p)
    return out


def rel(a, b):
    return max(float(np.max(np.abs(x - y)) / np.max(np.abs(y))) for x, y in zip(a, b))


@pytest.mark.parametrize("case", SGD_CASES, ids=[f"mu{c[0]}-d{c[1]}-nest{int(c[2])}-wd{c[3]}" for c in SGD_CASES])
def test_sgd_formulas_float64(case):
    mu, d, n, wd = case
    gs, lr_seq = grads(1, np.float64), lrs(0.05)
    p0, want, _ = torch_run(np.float64, lambda ps: torch.optim.SGD(ps, lr=0.05, momentum=mu, dampening=d, nesterov=n, weight_decay=wd),
                            gs, lr_seq, 1)
    got = replay_sgd(R.sgd64, p0, gs, lr_seq, mu, d, n, wd)
    assert rel(got, want) <= 1e-12


@pytest.mark.parametrize("case", ADAM_CASES, ids=[f"b{c[0][0]}-{c[0][1]}-wd{c[1]}-eps{c[2]}" for c in ADAM_CASES])
def test_adamw_formulas_float64(case):
    betas, wd, eps = case
    gs, lr_seq = grads(2, np.float64), lrs(1e-2)
    p0, want, opt = torch_run(np.float64, lambda ps: torch.optim.AdamW(ps, lr=1e-2, betas=betas, eps=eps, weight_decay=wd), gs, lr_seq, 2)
    got = replay_adamw(R.adamw64, p0, gs, lr_seq, betas, wd, eps, np.float64)
    assert rel(got, want) <= 1e-12


def ulps(a, b, p0):
    """|a - b| in units of the float32 spacing at the larger of |b| and the element's starting magnitude |p0| (an element that
    cancels to near 0 keeps the absolute error of the steps that led there)"""
    scale = np.maximum(np.abs(b), np.abs(p0))
    return np.abs(a.astype(np.float64) - b.astype(np.float64)) / np.spacing(scale).astype(np.float64)


ULP_BOUND = 64     # 20 steps of float32 rounding; torch's CPU kernels contract some products into FMAs (worst seen: 30)


def test_float32_replay_against_torch_float32():
    worst = {}
    for mu, d, n, wd in SGD_CASES:
        gs, lr_seq = grads(3, np.float32), lrs(0.05)
        p0, want, _ = torch_run(np.float32, lambda ps: torch.optim.SGD(ps, lr=0.05, momentum=mu, dampening=d, nesterov=n, weight_decay=wd),
                                gs, lr_seq, 3)
        got = replay_sgd(R.sgd32, p0, gs, lr_seq, mu, d, n, wd)
        worst[("sgd", mu, d, n, wd)] = max(float(np.max(ulps(x, y, z))) for x, y, z in zip(got, want, p0))
    for betas, wd, eps in ADAM_CASES:
        gs, lr_seq = grads(4, np.float32), lrs(1e-2)
        p0, want, _ = torch_run(np.float32, lambda ps: torch.optim.AdamW(ps, lr=1e-2, betas=betas, eps=eps, weight_decay=wd), gs, lr_seq, 4)
        got = replay_adamw(R.adamw32, p0, gs, lr_seq, betas, wd, eps, np.float32)
        worst[("adamw", betas, wd, eps)] = max(float(np.max(ulps(x, y, z))) for x, y, z in zip(got, want, p0))
    key = max(worst, key=worst.get)
    print(f"float32 replay vs torch float32 CPU optimizers: worst {worst[key]:.1f} ulp at {key}; "
          f"SGD worst {max(v for k, v in worst.items() if k[0] == 'sgd'):.1f}, AdamW worst {max(v for k, v in worst.items() if k[0] == 'adamw'):.1f}")
    assert worst[key] <= ULP_BOUND


def test_first_step_and_zero_decay_rules():
    """the clone on the first momentum step (no dampening), and wd = 0 skipping the decay term (0 * Inf would be NaN)"""
    p, g = np.array([np.inf, 1.0], np.float32), np.array([2.0, 4.0], np.float32)
    p1, b = R.sgd32(p, g, None, 0.5, 1, momentum=0.9, dampening=0.5)
    assert np.array_equal(b, g) and p1[0] == np.inf and p1[1] == np.float32(1.0) - np.float32(0.5) * np.float32(4.0)
    _, b2 = R.sgd32(p1, g, b, 0.5, 2, momentum=0.9, dampening=0.5)
    assert np.array_equal(b2, np.float32(0.9) * b + np.float32(0.5) * g)
    pa, m, v = R.adamw32(p, g, np.zeros(2, np.float32), np.zeros(2, np.float32), 1e-3, 1, wd=0.0)
    assert pa[0] == np.inf and np.isfinite(pa[1])


def test_resnet18_table():
    t = R.resnet18_tensors()
    assert len(t) == 62
    assert sum(int(np.prod(s)) for _, s, _ in t) == 11_689_512
    convs = [(n, s) for n, s, h in t if len(s) == 4 and h > 0]
    assert len(convs) == 20 and sum(1 for _, s in convs if s[3] % 8 == 0) == 19
