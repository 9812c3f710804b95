"""The depthwise convolution on the device (pcnn_dwconv_plan_create run by pcnn_conv_tc_fwd, pcnn_dwconv_dgrad, pcnn_dwconv_wgrad,
DepthwiseConvLayer): y and dx bit-identical to the float32 replays of tests/dwconv_ref.py (pinned to torch's CPU float64
conv2d(groups=C) by test_dwconv_cpu.py), dw exact on integer operands and within its error bound on random ones, buffers fully
written with nothing past them touched, exact adjointness, every refusal, plan refreshes by set_params and by the fused
optimizer, and torch's CUDA depthwise convolution on the same channels-last bf16 tensors recorded.

Error bound of dw (random operands): every partial sum is an fp32 sum of exact products, with n_acc additions on its longest path
(dwconv_info), so |dw - S| <= gamma A with gamma = n_acc u / (1 - n_acc u), u = 2^-24, S the exact sum and A the sum of |dy x|;
the test allows 2 n_acc u A."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dwconv_ref as DR
import pcnn_loader
from example_nets import DEV, NAN_BF16, MobileNetLite, host, train

pytestmark = pytest.mark.gpu

NAN_F32 = 0x7FC00000
TAIL = 64
U = 2.0 ** -24

CASES = [  # id, N, H, W, C, R, S, stride, pad_h, pad_w
    ("c1-3x3s1p1", 2, 9, 11, 1, 3, 3, 1, 1, 1),
    ("c3-5x5s2p2-odd", 2, 13, 11, 3, 5, 5, 2, 2, 2),
    ("c6-7x7s1p3", 2, 10, 12, 6, 7, 7, 1, 3, 3),
    ("c6-3x2s3-gaps", 3, 11, 10, 6, 3, 2, 3, 0, 0),
    ("c8-1x1s1", 2, 7, 9, 8, 1, 1, 1, 0, 0),
    ("c8-1x1s2", 2, 8, 9, 8, 1, 1, 2, 0, 0),
    ("c8-3x3s4p2-gaps", 2, 17, 14, 8, 3, 3, 4, 2, 2),
    ("c24-3x3s2p1", 2, 14, 14, 24, 3, 3, 2, 1, 1),
    ("c24-5x5s3p4", 2, 12, 13, 24, 5, 5, 3, 4, 4),
    ("c64-3x3s1p0", 2, 10, 9, 64, 3, 3, 1, 0, 0),
    ("c64-7x7s2p6", 1, 9, 9, 64, 7, 7, 2, 6, 6),
    ("c144-3x3s2p1-odd", 2, 15, 13, 144, 3, 3, 2, 1, 1),
    ("c144-3x2s1p1x0", 2, 8, 8, 144, 3, 2, 1, 1, 0),
    ("c256-5x5s1p2", 2, 7, 8, 256, 5, 5, 1, 2, 2),
    ("c320-3x3s1p1", 2, 7, 7, 320, 3, 3, 1, 1, 1),
    ("c320-7x7s4p3", 2, 16, 15, 320, 7, 7, 4, 3, 3),
    ("c960-3x3s1p1", 2, 7, 7, 960, 3, 3, 1, 1, 1),
    ("c960-5x5s2p2", 2, 8, 8, 960, 5, 5, 2, 2, 2),
    ("c3-1row-1x3s1p1", 3, 1, 9, 3, 1, 3, 1, 0, 1),
    ("c8-1row-3x3s1p1", 2, 1, 10, 8, 3, 3, 1, 1, 1),
    ("c64-1row-1x5s2p4", 2, 1, 12, 64, 1, 5, 2, 0, 4),
    ("c1-7x7s3p6", 2, 8, 9, 1, 7, 7, 3, 6, 6),
    ("c24-1x1s3", 2, 10, 10, 24, 1, 1, 3, 0, 0),
    ("mbv2-128x56x56x144-3x3s2", 128, 56, 56, 144, 3, 3, 2, 1, 1),
    ("effnet-128x28x28x240-5x5s1", 128, 28, 28, 240, 5, 5, 1, 2, 2),
]


_PK = pcnn_loader.load()              # the package's Python side only: the library is opened by the first call into it
bf, f32 = _PK.f32_to_bf16_bits, _PK.bf16_bits_to_f32


def same_or_nan(got, want):
    """bf16 bits: identical where want is a number; NaN (any payload) where want is NaN"""
    nan, gnan = (want & 0x7FFF) > 0x7F80, (got & 0x7FFF) > 0x7F80
    return np.array_equal(gnan, nan) and np.array_equal(got[~nan], want[~nan])


def special(rng, shape):
    x = rng.standard_normal(shape).astype(np.float32)
    flat = x.reshape(-1)
    for v, frac in ((np.nan, 0.01), (np.inf, 0.01), (-np.inf, 0.01), (0.0, 0.05), (-0.0, 0.05)):
        flat[rng.choice(flat.size, max(1, int(frac * flat.size)), replace=False)] = v
    return x


def padded(eng, bits, fill):
    """a device copy of `bits` followed by TAIL elements of `fill`"""
    flat = np.concatenate([np.ascontiguousarray(bits).reshape(-1), np.full(TAIL, fill, bits.dtype)])
    return eng.to_device(flat)


def out_buf(eng, n, dtype, fill):
    return eng.to_device(np.full(n + TAIL, fill, dtype))


def run_fwd(eng, plan, x_bits, out_shape):
    n = int(np.prod(out_shape))
    y = out_buf(eng, n, np.uint16, NAN_BF16)
    plan.fwd(padded(eng, x_bits, NAN_BF16), y)
    eng.sync()
    h = y.to_host()
    assert np.all(h[n:] == NAN_BF16)                                            # nothing past y is written
    return h[:n].reshape(out_shape)


def run_dgrad(eng, plan, dy_bits, x_shape):
    n = int(np.prod(x_shape))
    dx = out_buf(eng, n, np.uint16, NAN_BF16)
    eng.dwconv_dgrad(plan, padded(eng, dy_bits, NAN_BF16), dx)
    eng.sync()
    h = dx.to_host()
    assert np.all(h[n:] == NAN_BF16)
    return h[:n].reshape(x_shape)


def run_wgrad(eng, plan, x_bits, dy_bits, C, R, S):
    n = C * R * S
    dw = out_buf(eng, n, np.uint32, NAN_F32)
    eng.dwconv_wgrad(plan, padded(eng, x_bits, NAN_BF16), padded(eng, dy_bits, NAN_BF16), dw)
    eng.sync()
    h = dw.to_host()
    assert np.all(h[n:] == NAN_F32)
    return h[:n].view(np.float32).reshape(C, R, S)


def cuda_nchw(bits):
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).to(DEV).view(torch.bfloat16).permute(0, 3, 1, 2)


def host_bits(t):
    return t.permute(0, 2, 3, 1).contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_passes(eng, pkg, case):
    _, N, H, W, Cc, R, S, st, ph, pw = case
    info = pkg.dwconv_info(N, H, W, Cc, R, S, st, (ph, pw))
    P, Q = info["P"], info["Q"]
    assert (P, Q) == DR.out_size(H, W, R, S, st, ph, pw)
    rng = np.random.default_rng(sum(case[1:]))
    w = rng.standard_normal((Cc, R, S)).astype(np.float32)
    wq = f32(bf(w))
    b = rng.standard_normal(Cc).astype(np.float32)
    x_bits = bf(rng.standard_normal((N, H, W, Cc)).astype(np.float32))
    big = N * H * W * Cc > 10 ** 7
    # forward: with and without bias, no activation and ReLU, random and special values
    for bias in (None, b):
        for act in (0, 3):
            if big and (bias is None) != (act == 0):
                continue
            plan = pkg.DepthwiseConvPlan(eng, N, H, W, Cc, R, S, w, bias, act=act, stride=st, padding=(ph, pw))
            assert plan.out_shape == (N, P, Q, Cc)
            kinds = (("random", x_bits),) if big else (("random", x_bits), ("special", bf(special(rng, (N, H, W, Cc)))))
            for kind, xb in kinds:
                y = run_fwd(eng, plan, xb, (N, P, Q, Cc))
                want = bf(DR.fwd(f32(xb), wq, bias, st, ph, pw, act))
                assert same_or_nan(y, want), (kind, bias is not None, act, int(np.sum(y != want)))
                assert np.array_equal(run_fwd(eng, plan, xb, (N, P, Q, Cc)), y)                    # rerun
            plan.close()
    plan = pkg.DepthwiseConvPlan(eng, N, H, W, Cc, R, S, w, None, act=0, stride=st, padding=(ph, pw))
    # input gradient: random and special dy
    dy_bits = bf(rng.standard_normal((N, P, Q, Cc)).astype(np.float32))
    for kind, db in (("random", dy_bits),) + (() if big else (("special", bf(special(rng, (N, P, Q, Cc)))),)):
        dx = run_dgrad(eng, plan, db, (N, H, W, Cc))
        want, terms = DR.dgrad(f32(db), wq, H, W, st, ph, pw)
        assert same_or_nan(dx, bf(want)), (kind, int(np.sum(dx != bf(want))))
        assert np.all(dx[:, terms == 0] == 0)                                                      # +0 with no term
        assert np.array_equal(run_dgrad(eng, plan, db, (N, H, W, Cc)), dx)
    # weight gradient on random operands: within the bound
    dw = run_wgrad(eng, plan, x_bits, dy_bits, Cc, R, S)
    exact = DR.wgrad_f64(f32(x_bits), f32(dy_bits), R, S, st, ph, pw)
    A = DR.wgrad_abs_f64(f32(x_bits), f32(dy_bits), R, S, st, ph, pw)
    err = np.abs(dw.astype(np.float64) - exact)
    bound = 2 * info["n_acc"] * U * A
    assert np.all(err <= bound), float(np.max(err / np.maximum(bound, 1e-300)))
    assert np.array_equal(run_wgrad(eng, plan, x_bits, dy_bits, Cc, R, S).view(np.uint32), dw.view(np.uint32))   # rerun
    print(f"{case[0]}: dw worst error / bound = {float(np.max(err / np.maximum(bound, 1e-300))):.3f}, n_acc {info['n_acc']}, "
          f"ranges {info['ranges']}")
    plan.close()
    # integer operands: dw exact, and <y, dy> = <x, dx> = <w, dw> exactly
    wi = rng.integers(-2, 3, (Cc, R, S)).astype(np.float32)
    xi = bf(rng.integers(-2, 3, (N, H, W, Cc)).astype(np.float32))
    dyi = bf(rng.integers(-2, 3, (N, P, Q, Cc)).astype(np.float32))
    plan = pkg.DepthwiseConvPlan(eng, N, H, W, Cc, R, S, wi, None, act=0, stride=st, padding=(ph, pw))
    y = run_fwd(eng, plan, xi, (N, P, Q, Cc))
    dx = run_dgrad(eng, plan, dyi, (N, H, W, Cc))
    dw = run_wgrad(eng, plan, xi, dyi, Cc, R, S)
    assert np.array_equal(dw.astype(np.float64), DR.wgrad_f64(f32(xi), f32(dyi), R, S, st, ph, pw))
    lhs = np.sum(f32(y).astype(np.float64) * f32(dyi))
    assert lhs == np.sum(f32(dx).astype(np.float64) * f32(xi)) == np.sum(dw.astype(np.float64) * wi)
    plan.close()
    # torch's CUDA depthwise convolution on the same bf16 tensors, recorded
    plan = pkg.DepthwiseConvPlan(eng, N, H, W, Cc, R, S, w, None, act=0, stride=st, padding=(ph, pw))
    y = run_fwd(eng, plan, x_bits, (N, P, Q, Cc))
    dx = run_dgrad(eng, plan, dy_bits, (N, H, W, Cc))
    xt = cuda_nchw(x_bits).contiguous(memory_format=torch.channels_last)
    wt = torch.from_numpy(wq).to(DEV).to(torch.bfloat16)[:, None].contiguous(memory_format=torch.channels_last)
    ty = F.conv2d(xt, wt, None, st, (ph, pw), groups=Cc)
    gi, _, _ = torch.ops.aten.convolution_backward(cuda_nchw(dy_bits).contiguous(memory_format=torch.channels_last), xt, wt, None, [st, st],
                                                   [ph, pw], [1, 1], False, [0, 0], Cc, [True, False, False])
    print(f"{case[0]} vs torch CUDA: y bits differ on {int(np.sum(host_bits(ty) != y))} of {y.size}, "
          f"dx on {int(np.sum(host_bits(gi) != dx))} of {dx.size}")
    plan.close()


def test_layer_matches_the_calls(eng, pkg):
    """DepthwiseConvLayer with a bias and a ReLU: the bias/activation backward, then the gradients of the pre-activation"""
    N, H, W, Cc, R, S, st = 2, 9, 9, 24, 3, 3, 1
    rng = np.random.default_rng(3)
    w, b = rng.standard_normal((Cc, R, S)).astype(np.float32), rng.standard_normal(Cc).astype(np.float32)
    layer = pkg.DepthwiseConvLayer(eng, N, H, W, Cc, R, S, w, b, act=pkg.ACT_RELU, stride=st, padding=(1, 1))
    P, Q = layer.out_shape[1:3]
    x_bits = bf(rng.standard_normal((N, H, W, Cc)).astype(np.float32))
    dy_bits = bf(rng.standard_normal((N, P, Q, Cc)).astype(np.float32))
    x, y = eng.to_device(x_bits), eng.array((N, P, Q, Cc), np.uint16)
    dy, dx = eng.to_device(dy_bits), eng.array((N, H, W, Cc), np.uint16)
    layer.forward(x, y)
    layer.backward(y, dy, dx)
    eng.sync()
    wq = f32(bf(w))
    yv = DR.fwd(f32(x_bits), wq, b, st, 1, 1, 3)
    assert np.array_equal(y.to_host(), bf(yv))
    g = np.where(f32(bf(yv)) <= 0, np.float32(0), f32(dy_bits))
    assert np.array_equal(dy.to_host(), bf(g))                                                    # consumed in place
    assert np.array_equal(dx.to_host(), bf(DR.dgrad(g, wq, H, W, st, 1, 1)[0]))
    db = layer.db.to_host()
    assert np.allclose(db, g.astype(np.float64).sum(axis=(0, 1, 2)), rtol=1e-5, atol=1e-5)
    dw = layer.dw.to_host()
    assert np.allclose(dw, DR.wgrad_f64(f32(x_bits), g, R, S, st, 1, 1), rtol=1e-4, atol=1e-4)
    layer.close()


def test_refusals(eng, pkg):
    w = np.ones((8, 3, 3), np.float32)

    def refused(fn, words, *args, **kw):
        with pytest.raises(pkg.PcnnError) as e:
            fn(*args, **kw)
        assert words in e.value.msg, e.value.msg
        return e.value.msg

    # domain: the create call names itself and the rule
    m = refused(pkg.DepthwiseConvPlan, "1 <= stride <= 4", eng, 2, 8, 8, 8, 3, 3, w, stride=5)
    assert "pcnn_dwconv_plan_create" in m
    refused(pkg.DepthwiseConvPlan, "0 <= pad_h <= R - 1", eng, 2, 8, 8, 8, 3, 3, w, padding=(3, 0))
    refused(pkg.DepthwiseConvPlan, "1 <= R, S <= 7", eng, 2, 8, 8, 8, 8, 1, np.ones((8, 8, 1), np.float32))
    refused(pkg.DepthwiseConvPlan, "H + 2 pad_h >= R", eng, 2, 1, 8, 8, 3, 3, w)
    refused(pkg.DepthwiseConvPlan, "each must be >= 1", eng, 0, 8, 8, 8, 3, 3, w)
    refused(pkg.DepthwiseConvPlan, "act 1 (sigmoid) is not supported", eng, 2, 8, 8, 8, 3, 3, w, act=pkg.ACT_SIGMOID)
    refused(pkg.DepthwiseConvPlan, "act 2 is not 0", eng, 2, 8, 8, 8, 3, 3, w, act=2)
    L = pkg.lib()
    out = C.c_void_p()
    assert L.pcnn_dwconv_plan_create(eng.ctx, 2, 8, 8, 8, 3, 3, 1, 1, 1, 0, None, None, C.byref(out)) != 0
    assert "NULL" in L.pcnn_last_error_string().decode()
    plan = pkg.DepthwiseConvPlan(eng, 2, 8, 8, 8, 3, 3, w, padding=(1, 1))
    x, y = eng.array(2 * 8 * 8 * 8 + 64, np.uint16), eng.array(2 * 8 * 8 * 8 + 64, np.uint16)
    dw = eng.array(8 * 9 + 16)
    # NULL, alignment and overlap
    refused(eng.dwconv_wgrad, "NULL argument", plan, x, None, dw)
    refused(eng.dwconv_dgrad, "NULL argument", plan, None, x)
    refused(plan.fwd, "16-byte aligned", x.ptr + 2, y)
    refused(plan.fwd, "16-byte aligned", x, y.ptr + 2)
    refused(plan.fwd, "must not share memory", x, x.ptr + 16)
    refused(eng.dwconv_dgrad, "16-byte aligned", plan, x.ptr + 2, y)
    refused(eng.dwconv_dgrad, "must not share memory", plan, x, x.ptr + 32)
    refused(eng.dwconv_wgrad, "16-byte aligned", plan, x, y, dw.ptr + 4)
    refused(eng.dwconv_wgrad, "16-byte aligned", plan, x.ptr + 2, y, dw)
    # a plan of another kind
    lin = pkg.LinearPlan(eng, 2, 1, 1, 8, 8, np.ones((8, 8), np.float32))
    conv = pkg.WideConvPlan(eng, 2, 8, 8, 64, 64, 3, 3, np.ones((64, 3, 3, 64), np.float32))
    for other in (lin, conv):
        refused(eng.dwconv_wgrad, "was not made by pcnn_dwconv_plan_create", other, x, y, dw)
        refused(eng.dwconv_dgrad, "was not made by pcnn_dwconv_plan_create", other, x, y)
    refused(eng.linear_dgrad, "was not made by pcnn_linear_plan_create", plan, x, y)
    # a bias for a plan created without one
    refused(plan.set_params, "created without one", None, eng.array(8))
    for p in (plan, lin, conv):
        p.close()


def test_set_params_refresh(eng, pkg):
    N, H, W, Cc, R, S = 4, 12, 12, 64, 5, 5
    rng = np.random.default_rng(11)
    w1, w2 = (rng.standard_normal((Cc, R, S)).astype(np.float32) for _ in range(2))
    b1, b2 = (rng.standard_normal(Cc).astype(np.float32) for _ in range(2))
    x_bits = bf(rng.standard_normal((N, H, W, Cc)).astype(np.float32))
    dy_bits = bf(rng.standard_normal((N, H, W, Cc)).astype(np.float32))
    fresh = {}
    for k, (w, b) in {1: (w1, b1), 2: (w2, b2)}.items():
        p = pkg.DepthwiseConvPlan(eng, N, H, W, Cc, R, S, w, b, act=3, padding=(2, 2))
        fresh[k] = (run_fwd(eng, p, x_bits, (N, H, W, Cc)), run_dgrad(eng, p, dy_bits, (N, H, W, Cc)))
        p.close()
    plan = pkg.DepthwiseConvPlan(eng, N, H, W, Cc, R, S, w1, b1, act=3, padding=(2, 2))
    d1w, d1b, d2w, d2b = (eng.to_device(a) for a in (w1, b1, w2, b2))
    x = eng.to_device(x_bits)
    ys = [eng.array((N, H, W, Cc), np.uint16) for _ in range(3)]
    plan.fwd(x, ys[0])                                 # fwd -> set -> fwd -> set -> fwd with no synchronisation
    plan.set_params(d2w, d2b)
    plan.fwd(x, ys[1])
    plan.set_params(d1w, d1b)
    plan.fwd(x, ys[2])
    eng.sync()
    assert np.array_equal(ys[0].to_host(), fresh[1][0]) and np.array_equal(ys[2].to_host(), fresh[1][0])
    assert np.array_equal(ys[1].to_host(), fresh[2][0])
    plan.set_params(d2w, d2b)
    assert np.array_equal(run_dgrad(eng, plan, dy_bits, (N, H, W, Cc)), fresh[2][1])
    plan.close()


def _step(eng, layer, x, dy_bits):
    N, H, W, Cc, R, S = layer.shape
    y = eng.array(layer.out_shape, np.uint16)
    layer.forward(x, y)
    layer.backward(y, eng.to_device(dy_bits), eng.array((N, H, W, Cc), np.uint16))


@pytest.mark.parametrize("Cc", [144, 6])
def test_optimizer_refreshes_the_plan(eng, pkg, Cc):
    """A depthwise layer in a FusedOptimizer table: after each step the forward and the input gradient are bit-identical to those
    of a plan created from the new master"""
    N, H, W, R, S, st = 4, 14, 14, 3, 3, 2
    rng = np.random.default_rng(Cc)
    w, b = rng.standard_normal((Cc, R, S)).astype(np.float32), rng.standard_normal(Cc).astype(np.float32)
    layer = pkg.DepthwiseConvLayer(eng, N, H, W, Cc, R, S, w, b, act=3, stride=st, padding=(1, 1))
    P, Q = layer.out_shape[1:3]
    x_bits = bf(rng.standard_normal((N, H, W, Cc)).astype(np.float32))
    x = eng.to_device(x_bits)
    for opt in (pkg.SGD(eng, [layer], momentum=0.9, nesterov=True, weight_decay=1e-2), pkg.AdamW(eng, [layer], weight_decay=0.05)):
        for _ in range(3):
            _step(eng, layer, x, bf(rng.standard_normal((N, P, Q, Cc)).astype(np.float32)))
            opt.step(0.05)
        eng.sync()
        wm, bm = layer.params()
        fresh = pkg.DepthwiseConvPlan(eng, N, H, W, Cc, R, S, wm, bm, act=3, stride=st, padding=(1, 1))
        dy_bits = bf(rng.standard_normal((N, P, Q, Cc)).astype(np.float32))
        assert np.array_equal(run_fwd(eng, layer.plan, x_bits, layer.out_shape), run_fwd(eng, fresh, x_bits, layer.out_shape))
        assert np.array_equal(run_dgrad(eng, layer.plan, dy_bits, (N, H, W, Cc)), run_dgrad(eng, fresh, dy_bits, (N, H, W, Cc)))
        fresh.close()
        opt.close()
    layer.close()


def test_sgd_step_matches_layer_sgd(eng, pkg):
    N, H, W, Cc, R, S = 4, 10, 10, 64, 3, 3
    rng = np.random.default_rng(5)
    w, b = rng.standard_normal((Cc, R, S)).astype(np.float32), rng.standard_normal(Cc).astype(np.float32)
    a = pkg.DepthwiseConvLayer(eng, N, H, W, Cc, R, S, w, b, act=3, padding=(1, 1))
    c = pkg.DepthwiseConvLayer(eng, N, H, W, Cc, R, S, w, b, act=3, padding=(1, 1))
    x_bits = bf(rng.standard_normal((N, H, W, Cc)).astype(np.float32))
    x = eng.to_device(x_bits)
    opt = pkg.SGD(eng, [a])
    for _ in range(3):
        dy_bits = bf(rng.standard_normal((N, H, W, Cc)).astype(np.float32))
        _step(eng, a, x, dy_bits)
        _step(eng, c, x, dy_bits)
        opt.step(0.1)
        c.sgd(0.1)
    eng.sync()
    for u, v in zip(a.params(), c.params()):
        assert np.array_equal(u.view(np.uint32), v.view(np.uint32))
    assert np.array_equal(run_fwd(eng, a.plan, x_bits, a.out_shape), run_fwd(eng, c.plan, x_bits, c.out_shape))
    opt.close()
    a.close()
    c.close()


# ------------------------------------------------------------------------------------------------ end to end
ACC_MIN = 0.88          # a float32 torch CPU replica of this network, initialisation and step reaches 0.934 (DESIGN 3.18)


def test_mobilenet_mnist(eng, pkg, golden):
    """In each of the first 5 steps both depthwise layers' y and dx are bit-exact against the replays on the device's own tensors
    and dw lies within its bound.  A fresh run reproduces the parameters after 5 steps bit for bit.  After EPOCHS epochs over the
    1024 training digits the mean loss has fallen, and test accuracy on the 256 test digits, evaluated with the running statistics,
    exceeds ACC_MIN."""

    def check_step(net, it, x, labels):
        net.forward(x, labels)
        net.backward()
        eng.sync()
        for layer, x, y, dy, dx in ((net.d1, net.ze1, net.yd1, net.dyd1, net.dze1), (net.d2, net.ze2, net.yd2, net.dyd2, net.dze2)):
            N, H, W, Cc, R, S = layer.shape
            wq = f32(bf(layer.params()[0]))
            xv, dyv = f32(host(x)).reshape(N, H, W, Cc), f32(host(dy)).reshape(layer.out_shape)
            assert np.array_equal(host(y).reshape(layer.out_shape), bf(DR.fwd(xv, wq, None, layer.stride, 1, 1))), it
            assert np.array_equal(host(dx).reshape(N, H, W, Cc), bf(DR.dgrad(dyv, wq, H, W, layer.stride, 1, 1)[0])), it
            err = np.abs(layer.dw.to_host().astype(np.float64) - DR.wgrad_f64(xv, dyv, R, S, layer.stride, 1, 1))
            assert np.all(err <= 2 * layer.info["n_acc"] * U * DR.wgrad_abs_f64(xv, dyv, R, S, layer.stride, 1, 1)), it

    ep_loss, acc, _ = train(eng, pkg, golden, lambda: MobileNetLite(eng, pkg, MobileNetLite.init_params()), MobileNetLite.EPOCHS,
                            check_step=check_step)
    print(f"MobileNet-style network: mean loss by epoch {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}; test accuracy {acc:.4f} (threshold {ACC_MIN})")
    assert np.isfinite(ep_loss).all() and ep_loss[-1] < ep_loss[0]
    assert acc > ACC_MIN
