"""The grouped convolution on the device (pcnn_gconv_plan_create run by pcnn_conv_tc_fwd, pcnn_gconv_dgrad, pcnn_gconv_wgrad,
GroupedConvLayer): y and dx bit-identical to the float32 replays of tests/gconv_ref.py (pinned to torch's CPU float64
conv2d(groups=G) by test_gconv_cpu.py), dw exact on integer operands and within its error bound on random ones, buffers fully
written with nothing past them touched, exact adjointness, every refusal, plan refreshes by set_params and by the fused
optimizer, torch's CUDA grouped convolution on the same channels-last bf16 tensors recorded, and a ResNeXt-style network trained
on the golden MNIST subset.

Error bound of dw (random operands): every partial sum is an fp32 sum of exact products, with n_acc additions on its longest path
(gconv_info), so |dw - S| <= gamma A with gamma = n_acc u / (1 - n_acc u), u = 2^-24, S the exact sum and A the sum of |dy x|;
the test allows 2 n_acc u A."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gconv_ref as GR
import pcnn_loader
from example_nets import DEV, NAN_BF16, ResNeXtLite, host, train

pytestmark = pytest.mark.gpu

NAN_F32 = 0x7FC00000
TAIL = 64
U = 2.0 ** -24

CASES = [  # id, N, H, W, C, K, G, R, S, stride, pad_h, pad_w
    ("cg1kg2-mult-3x3s1p1", 2, 9, 11, 4, 8, 4, 3, 3, 1, 1, 1),
    ("cg2kg3-5x5s2p2-odd", 2, 13, 11, 6, 9, 3, 5, 5, 2, 2, 2),
    ("cg4kg2-7x7s1p3", 2, 10, 12, 8, 4, 2, 7, 7, 1, 3, 3),
    ("cg4kg8-3x2s3-gaps", 3, 11, 10, 8, 16, 2, 3, 2, 3, 0, 0),
    ("cg8kg4-1x1s1", 2, 7, 9, 16, 8, 2, 1, 1, 1, 0, 0),
    ("cg8kg16-1x1s2", 2, 8, 9, 16, 32, 2, 1, 1, 2, 0, 0),
    ("cg8kg4-3x3s4p2-gaps", 2, 17, 14, 32, 16, 4, 3, 3, 4, 2, 2),
    ("cg16kg32-3x3s2p1", 2, 14, 14, 32, 64, 2, 3, 3, 2, 1, 1),
    ("cg16kg4-5x5s3p4", 2, 12, 13, 32, 8, 2, 5, 5, 3, 4, 4),
    ("cg32kg16-3x3s1p0", 2, 10, 9, 64, 32, 2, 3, 3, 1, 0, 0),
    ("cg64kg32-3x3s1p1", 2, 7, 7, 128, 64, 2, 3, 3, 1, 1, 1),
    ("cg64kg64-1x1s1", 2, 7, 8, 128, 128, 2, 1, 1, 1, 0, 0),
    ("cg3kg3-1row-1x3s1p1", 3, 1, 9, 6, 6, 2, 1, 3, 1, 0, 1),
    ("cg2kg1-1row-3x3s1p1", 2, 1, 10, 8, 4, 4, 3, 3, 1, 1, 1),
    ("cg6kg1-7x7s3p6", 2, 8, 9, 12, 2, 2, 7, 7, 3, 6, 6),
    ("cg4kg4-1x1s3", 2, 10, 10, 16, 16, 4, 1, 1, 3, 0, 0),
    ("cg2kg4-shuffle-1x1", 2, 9, 9, 24, 48, 12, 1, 1, 1, 0, 0),
    ("cg1kg2-slices-3x3s1p1", 2, 6, 6, 512, 1024, 512, 3, 3, 1, 1, 1),
    ("cg16kg16-regnet-slices", 2, 7, 7, 384, 384, 24, 3, 3, 1, 1, 1),
    ("resnext-128x56x56x128-g32", 128, 56, 56, 128, 128, 32, 3, 3, 1, 1, 1),
    ("resnext-128x28x28x256-g32-s2", 128, 28, 28, 256, 256, 32, 3, 3, 2, 1, 1),
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
    eng.gconv_dgrad(plan, padded(eng, dy_bits, NAN_BF16), dx)
    eng.sync()
    h = dx.to_host()
    assert np.all(h[n:] == NAN_BF16)
    return h[:n].reshape(x_shape)


def run_wgrad(eng, plan, x_bits, dy_bits, w_shape):
    n = int(np.prod(w_shape))
    dw = out_buf(eng, n, np.uint32, NAN_F32)
    eng.gconv_wgrad(plan, padded(eng, x_bits, NAN_BF16), padded(eng, dy_bits, NAN_BF16), dw)
    eng.sync()
    h = dw.to_host()
    assert np.all(h[n:] == NAN_F32)
    return h[:n].view(np.float32).reshape(w_shape)


def cuda_nchw(bits):
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).to(DEV).view(torch.bfloat16).permute(0, 3, 1, 2)


def host_bits(t):
    return t.permute(0, 2, 3, 1).contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_passes(eng, pkg, case):
    _, N, H, W, Cc, K, G, R, S, st, ph, pw = case
    info = pkg.gconv_info(N, H, W, Cc, K, G, R, S, st, (ph, pw))
    P, Q, Cg = info["P"], info["Q"], info["Cg"]
    assert (P, Q) == GR.out_size(H, W, R, S, st, ph, pw)
    rng = np.random.default_rng(sum(case[1:]))
    w = rng.standard_normal((K, R, S, Cg)).astype(np.float32)
    wq = f32(bf(w))
    b = rng.standard_normal(K).astype(np.float32)
    x_bits = bf(rng.standard_normal((N, H, W, Cc)).astype(np.float32))
    big = N * H * W * Cc > 10 ** 7
    # forward: with and without bias, no activation and ReLU, random and special values
    for bias in (None, b):
        for act in (0, 3):
            if big and (bias is None) != (act == 0):
                continue
            plan = pkg.GroupedConvPlan(eng, N, H, W, Cc, K, G, R, S, w, bias, act=act, stride=st, padding=(ph, pw))
            assert plan.out_shape == (N, P, Q, K)
            kinds = (("random", x_bits),) if big else (("random", x_bits), ("special", bf(special(rng, (N, H, W, Cc)))))
            for kind, xb in kinds:
                y = run_fwd(eng, plan, xb, (N, P, Q, K))
                want = bf(GR.fwd(f32(xb), wq, G, bias, st, ph, pw, act))
                assert same_or_nan(y, want), (kind, bias is not None, act, int(np.sum(y != want)))
                assert np.array_equal(run_fwd(eng, plan, xb, (N, P, Q, K)), y)                     # rerun
            plan.close()
    plan = pkg.GroupedConvPlan(eng, N, H, W, Cc, K, G, R, S, w, None, act=0, stride=st, padding=(ph, pw))
    # input gradient: random and special dy
    dy_bits = bf(rng.standard_normal((N, P, Q, K)).astype(np.float32))
    for kind, db in (("random", dy_bits),) + (() if big else (("special", bf(special(rng, (N, P, Q, K)))),)):
        dx = run_dgrad(eng, plan, db, (N, H, W, Cc))
        want, terms = GR.dgrad(f32(db), wq, G, H, W, st, ph, pw)
        assert same_or_nan(dx, bf(want)), (kind, int(np.sum(dx != bf(want))))
        assert np.all(dx[:, terms == 0] == 0)                                                      # +0 with no term
        assert np.array_equal(run_dgrad(eng, plan, db, (N, H, W, Cc)), dx)
    # weight gradient on random operands: within the bound
    dw = run_wgrad(eng, plan, x_bits, dy_bits, (K, R, S, Cg))
    exact = GR.wgrad_f64(f32(x_bits), f32(dy_bits), G, R, S, st, ph, pw)
    A = GR.wgrad_abs_f64(f32(x_bits), f32(dy_bits), G, R, S, st, ph, pw)
    err = np.abs(dw.astype(np.float64) - exact)
    bound = 2 * info["n_acc"] * U * A
    assert np.all(err <= bound), float(np.max(err / np.maximum(bound, 1e-300)))
    assert np.array_equal(run_wgrad(eng, plan, x_bits, dy_bits, (K, R, S, Cg)).view(np.uint32), dw.view(np.uint32))   # rerun
    print(f"{case[0]}: dw worst error / bound = {float(np.max(err / np.maximum(bound, 1e-300))):.3f}, n_acc {info['n_acc']}, "
          f"ranges {info['ranges']}, vec {info['vec']}, kt {info['kt']}")
    plan.close()
    # integer operands: dw exact, and <y, dy> = <x, dx> = <w, dw> exactly
    wi = rng.integers(-2, 3, (K, R, S, Cg)).astype(np.float32)
    xi = bf(rng.integers(-2, 3, (N, H, W, Cc)).astype(np.float32))
    dyi = bf(rng.integers(-2, 3, (N, P, Q, K)).astype(np.float32))
    plan = pkg.GroupedConvPlan(eng, N, H, W, Cc, K, G, R, S, wi, None, act=0, stride=st, padding=(ph, pw))
    y = run_fwd(eng, plan, xi, (N, P, Q, K))
    dx = run_dgrad(eng, plan, dyi, (N, H, W, Cc))
    dw = run_wgrad(eng, plan, xi, dyi, (K, R, S, Cg))
    assert np.array_equal(dw.astype(np.float64), GR.wgrad_f64(f32(xi), f32(dyi), G, R, S, st, ph, pw))
    lhs = np.sum(f32(y).astype(np.float64) * f32(dyi))
    assert lhs == np.sum(f32(dx).astype(np.float64) * f32(xi)) == np.sum(dw.astype(np.float64) * wi)
    plan.close()
    # torch's CUDA grouped convolution on the same bf16 tensors, recorded
    plan = pkg.GroupedConvPlan(eng, N, H, W, Cc, K, G, R, S, w, None, act=0, stride=st, padding=(ph, pw))
    y = run_fwd(eng, plan, x_bits, (N, P, Q, K))
    dx = run_dgrad(eng, plan, dy_bits, (N, H, W, Cc))
    xt = cuda_nchw(x_bits).contiguous(memory_format=torch.channels_last)
    wt = torch.from_numpy(wq).to(DEV).to(torch.bfloat16).permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
    ty = F.conv2d(xt, wt, None, st, (ph, pw), groups=G)
    gi, _, _ = torch.ops.aten.convolution_backward(cuda_nchw(dy_bits).contiguous(memory_format=torch.channels_last), xt, wt, None, [st, st],
                                                   [ph, pw], [1, 1], False, [0, 0], G, [True, False, False])
    print(f"{case[0]} vs torch CUDA: y bits differ on {int(np.sum(host_bits(ty) != y))} of {y.size}, "
          f"dx on {int(np.sum(host_bits(gi) != dx))} of {dx.size}")
    plan.close()


def test_layer_matches_the_calls(eng, pkg):
    """GroupedConvLayer with a bias and a ReLU: the bias/activation backward, then the gradients of the pre-activation"""
    N, H, W, Cc, K, G, R, S, st = 2, 9, 9, 32, 48, 8, 3, 3, 1
    rng = np.random.default_rng(3)
    w, b = rng.standard_normal((K, R, S, Cc // G)).astype(np.float32), rng.standard_normal(K).astype(np.float32)
    layer = pkg.GroupedConvLayer(eng, N, H, W, Cc, K, G, R, S, w, b, act=pkg.ACT_RELU, stride=st, padding=(1, 1))
    P, Q = layer.out_shape[1:3]
    x_bits = bf(rng.standard_normal((N, H, W, Cc)).astype(np.float32))
    dy_bits = bf(rng.standard_normal((N, P, Q, K)).astype(np.float32))
    x, y = eng.to_device(x_bits), eng.array((N, P, Q, K), np.uint16)
    dy, dx = eng.to_device(dy_bits), eng.array((N, H, W, Cc), np.uint16)
    layer.forward(x, y)
    layer.backward(y, dy, dx)
    eng.sync()
    wq = f32(bf(w))
    yv = GR.fwd(f32(x_bits), wq, G, b, st, 1, 1, 3)
    assert np.array_equal(y.to_host(), bf(yv))
    g = np.where(f32(bf(yv)) <= 0, np.float32(0), f32(dy_bits))
    assert np.array_equal(dy.to_host(), bf(g))                                                    # consumed in place
    assert np.array_equal(dx.to_host(), bf(GR.dgrad(g, wq, G, H, W, st, 1, 1)[0]))
    assert np.allclose(layer.db.to_host(), g.astype(np.float64).sum(axis=(0, 1, 2)), rtol=1e-5, atol=1e-5)
    assert np.allclose(layer.dw.to_host(), GR.wgrad_f64(f32(x_bits), g, G, R, S, st, 1, 1), rtol=1e-4, atol=1e-4)
    layer.close()


def test_refusals(eng, pkg):
    w = np.ones((16, 3, 3, 4), np.float32)

    def refused(fn, words, *args, **kw):
        with pytest.raises(pkg.PcnnError) as e:
            fn(*args, **kw)
        assert words in e.value.msg, e.value.msg
        return e.value.msg

    # domain: the create call names itself and the rule
    m = refused(pkg.GroupedConvPlan, "1 <= stride <= 4", eng, 2, 8, 8, 8, 16, 2, 3, 3, w, stride=5)
    assert "pcnn_gconv_plan_create" in m
    refused(pkg.GroupedConvPlan, "0 <= pad_h <= R - 1", eng, 2, 8, 8, 8, 16, 2, 3, 3, w, padding=(3, 0))
    refused(pkg.GroupedConvPlan, "1 <= R, S <= 7", eng, 2, 8, 8, 8, 16, 2, 8, 1, np.ones((16, 8, 1, 4), np.float32))
    refused(pkg.GroupedConvPlan, "H + 2 pad_h >= R", eng, 2, 1, 8, 8, 16, 2, 3, 3, w)
    refused(pkg.GroupedConvPlan, "each must be >= 1", eng, 0, 8, 8, 8, 16, 2, 3, 3, w)
    refused(pkg.GroupedConvPlan, "groups = 1 is a dense convolution", eng, 2, 8, 8, 4, 16, 1, 3, 3, w)
    refused(pkg.GroupedConvPlan, "use pcnn_dwconv_plan_create", eng, 2, 8, 8, 8, 8, 8, 3, 3, np.ones((8, 3, 3, 1), np.float32))
    refused(pkg.GroupedConvPlan, "C % G == 0 and K % G == 0", eng, 2, 8, 8, 8, 18, 4, 3, 3, np.ones((18, 3, 3, 2), np.float32))
    refused(pkg.GroupedConvPlan, "Kg Cg R S <= 36864", eng, 2, 8, 8, 256, 256, 2, 3, 3, np.ones((256, 3, 3, 128), np.float32))
    refused(pkg.GroupedConvPlan, "act 1 (sigmoid) is not supported", eng, 2, 8, 8, 8, 16, 2, 3, 3, w, act=pkg.ACT_SIGMOID)
    refused(pkg.GroupedConvPlan, "act 2 is not 0", eng, 2, 8, 8, 8, 16, 2, 3, 3, w, act=2)
    L = pkg.lib()
    out = C.c_void_p()
    assert L.pcnn_gconv_plan_create(eng.ctx, 2, 8, 8, 8, 16, 2, 3, 3, 1, 1, 1, 0, None, None, C.byref(out)) != 0
    assert "NULL" in L.pcnn_last_error_string().decode()
    plan = pkg.GroupedConvPlan(eng, 2, 8, 8, 8, 16, 2, 3, 3, w, padding=(1, 1))
    x, y = eng.array(2 * 8 * 8 * 16 + 64, np.uint16), eng.array(2 * 8 * 8 * 16 + 64, np.uint16)
    dw = eng.array(16 * 9 * 4 + 16)
    # NULL, alignment and overlap
    refused(eng.gconv_wgrad, "NULL argument", plan, x, None, dw)
    refused(eng.gconv_dgrad, "NULL argument", plan, None, x)
    refused(plan.fwd, "16-byte aligned", x.ptr + 2, y)
    refused(plan.fwd, "16-byte aligned", x, y.ptr + 2)
    refused(plan.fwd, "must not share memory", x, x.ptr + 16)
    refused(eng.gconv_dgrad, "16-byte aligned", plan, x.ptr + 2, y)
    refused(eng.gconv_dgrad, "must not share memory", plan, x, x.ptr + 32)
    refused(eng.gconv_wgrad, "16-byte aligned", plan, x, y, dw.ptr + 4)
    refused(eng.gconv_wgrad, "16-byte aligned", plan, x.ptr + 2, y, dw)
    refused(eng.gconv_wgrad, "must not share memory", plan, x, y, x.ptr + 16)
    # plans of the other kinds, both ways
    lin = pkg.LinearPlan(eng, 2, 1, 1, 8, 8, np.ones((8, 8), np.float32))
    conv = pkg.WideConvPlan(eng, 2, 8, 8, 64, 64, 3, 3, np.ones((64, 3, 3, 64), np.float32))
    dwp = pkg.DepthwiseConvPlan(eng, 2, 8, 8, 8, 3, 3, np.ones((8, 3, 3), np.float32), padding=(1, 1))
    narrow = pkg.ConvPlan(eng, 2, 8, 8, 1, 8, 3, 3, np.ones((8, 3, 3, 1), np.float32))
    for other in (lin, conv, dwp, narrow):
        refused(eng.gconv_wgrad, "was not made by pcnn_gconv_plan_create", other, x, y, dw)
        refused(eng.gconv_dgrad, "was not made by pcnn_gconv_plan_create", other, x, y)
    refused(eng.linear_dgrad, "was not made by pcnn_linear_plan_create", plan, x, y)
    refused(eng.linear_wgrad, "was not made by pcnn_linear_plan_create", plan, x, y, dw)
    refused(eng.dwconv_dgrad, "was not made by pcnn_dwconv_plan_create", plan, x, y)
    refused(eng.dwconv_wgrad, "was not made by pcnn_dwconv_plan_create", plan, x, y, dw)
    # a bias for a plan created without one
    refused(plan.set_params, "created without one", None, eng.array(16))
    for p in (plan, lin, conv, dwp, narrow):
        p.close()


def test_set_params_refresh(eng, pkg):
    N, H, W, Cc, K, G, R, S = 4, 12, 12, 64, 32, 8, 5, 5
    rng = np.random.default_rng(11)
    w1, w2 = (rng.standard_normal((K, R, S, Cc // G)).astype(np.float32) for _ in range(2))
    b1, b2 = (rng.standard_normal(K).astype(np.float32) for _ in range(2))
    x_bits = bf(rng.standard_normal((N, H, W, Cc)).astype(np.float32))
    dy_bits = bf(rng.standard_normal((N, H, W, K)).astype(np.float32))
    fresh = {}
    for k, (w, b) in {1: (w1, b1), 2: (w2, b2)}.items():
        p = pkg.GroupedConvPlan(eng, N, H, W, Cc, K, G, R, S, w, b, act=3, padding=(2, 2))
        fresh[k] = (run_fwd(eng, p, x_bits, (N, H, W, K)), run_dgrad(eng, p, dy_bits, (N, H, W, Cc)))
        p.close()
    plan = pkg.GroupedConvPlan(eng, N, H, W, Cc, K, G, R, S, w1, b1, act=3, padding=(2, 2))
    d1w, d1b, d2w, d2b = (eng.to_device(a) for a in (w1, b1, w2, b2))
    x = eng.to_device(x_bits)
    ys = [eng.array((N, H, W, K), np.uint16) for _ in range(3)]
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
    N, H, W, Cc = layer.shape[:4]
    y = eng.array(layer.out_shape, np.uint16)
    layer.forward(x, y)
    layer.backward(y, eng.to_device(dy_bits), eng.array((N, H, W, Cc), np.uint16))


@pytest.mark.parametrize("shape", [(64, 64, 16), (12, 24, 6)], ids=["cg4kg4", "cg2kg4"])
def test_optimizer_refreshes_the_plan(eng, pkg, shape):
    """A grouped layer in a FusedOptimizer table: after each step the forward and the input gradient are bit-identical to those
    of a plan created from the new master"""
    Cc, K, G = shape
    N, H, W, R, S, st = 4, 14, 14, 3, 3, 2
    rng = np.random.default_rng(Cc)
    w, b = rng.standard_normal((K, R, S, Cc // G)).astype(np.float32), rng.standard_normal(K).astype(np.float32)
    layer = pkg.GroupedConvLayer(eng, N, H, W, Cc, K, G, R, S, w, b, act=3, stride=st, padding=(1, 1))
    P, Q = layer.out_shape[1:3]
    x_bits = bf(rng.standard_normal((N, H, W, Cc)).astype(np.float32))
    x = eng.to_device(x_bits)
    for opt in (pkg.SGD(eng, [layer], momentum=0.9, nesterov=True, weight_decay=1e-2), pkg.AdamW(eng, [layer], weight_decay=0.05)):
        for _ in range(3):
            _step(eng, layer, x, bf(rng.standard_normal((N, P, Q, K)).astype(np.float32)))
            opt.step(0.05)
        eng.sync()
        wm, bm = layer.params()
        fresh = pkg.GroupedConvPlan(eng, N, H, W, Cc, K, G, R, S, wm, bm, act=3, stride=st, padding=(1, 1))
        dy_bits = bf(rng.standard_normal((N, P, Q, K)).astype(np.float32))
        assert np.array_equal(run_fwd(eng, layer.plan, x_bits, layer.out_shape), run_fwd(eng, fresh, x_bits, layer.out_shape))
        assert np.array_equal(run_dgrad(eng, layer.plan, dy_bits, (N, H, W, Cc)), run_dgrad(eng, fresh, dy_bits, (N, H, W, Cc)))
        fresh.close()
        opt.close()
    layer.close()


def test_sgd_step_matches_layer_sgd(eng, pkg):
    N, H, W, Cc, K, G, R, S = 4, 10, 10, 64, 64, 8, 3, 3
    rng = np.random.default_rng(5)
    w, b = rng.standard_normal((K, R, S, Cc // G)).astype(np.float32), rng.standard_normal(K).astype(np.float32)
    a = pkg.GroupedConvLayer(eng, N, H, W, Cc, K, G, R, S, w, b, act=3, padding=(1, 1))
    c = pkg.GroupedConvLayer(eng, N, H, W, Cc, K, G, R, S, w, b, act=3, padding=(1, 1))
    x_bits = bf(rng.standard_normal((N, H, W, Cc)).astype(np.float32))
    x = eng.to_device(x_bits)
    opt = pkg.SGD(eng, [a])
    for _ in range(3):
        dy_bits = bf(rng.standard_normal((N, H, W, K)).astype(np.float32))
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
ACC_MIN = 0.85          # below the accuracy of the float32 torch CPU replica, scripts/resnext_replica.py (DESIGN 3.21)


def test_resnext_mnist(eng, pkg, golden):
    """In each of the first 5 steps both grouped layers' y and dx are bit-exact against the replays on the device's own tensors
    and dw lies within its bound.  A fresh run reproduces the parameters after 5 steps bit for bit.  After EPOCHS epochs over the
    1024 training digits the mean loss has fallen, and test accuracy on the 256 test digits, evaluated with the running statistics,
    exceeds ACC_MIN."""

    def check_step(net, it, x, labels):
        net.forward(x, labels)
        net.backward()
        eng.sync()
        for layer, x, y, dy, dx in ((net.g1, net.ze1, net.yg1, net.dyg1, net.dze1), (net.g2, net.ze2, net.yg2, net.dyg2, net.dze2)):
            N, H, W, Cc, K, G, R, S = layer.shape
            wq = f32(bf(layer.params()[0]))
            xv, dyv = f32(host(x)).reshape(N, H, W, Cc), f32(host(dy)).reshape(layer.out_shape)
            assert np.array_equal(host(y).reshape(layer.out_shape), bf(GR.fwd(xv, wq, G, None, layer.stride, 1, 1))), it
            assert np.array_equal(host(dx).reshape(N, H, W, Cc), bf(GR.dgrad(dyv, wq, G, H, W, layer.stride, 1, 1)[0])), it
            err = np.abs(layer.dw.to_host().astype(np.float64) - GR.wgrad_f64(xv, dyv, G, R, S, layer.stride, 1, 1))
            assert np.all(err <= 2 * layer.info["n_acc"] * U * GR.wgrad_abs_f64(xv, dyv, G, R, S, layer.stride, 1, 1)), it

    ep_loss, acc, _ = train(eng, pkg, golden, lambda: ResNeXtLite(eng, pkg, ResNeXtLite.init_params()), ResNeXtLite.EPOCHS,
                            check_step=check_step)
    print(f"ResNeXt-style network: mean loss by epoch {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}; test accuracy {acc:.4f} (threshold {ACC_MIN})")
    assert np.isfinite(ep_loss).all() and ep_loss[-1] < ep_loss[0]
    assert acc > ACC_MIN
