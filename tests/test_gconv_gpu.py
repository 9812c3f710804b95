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

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
NAN_BF16 = 0x7FC0
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
NB = 128
LR_STEP = 0.2
EPOCHS = 40
ACC_MIN = 0.85          # below the accuracy of the float32 torch CPU replica, scripts/resnext_replica.py (DESIGN 3.21)


def init_params(seed=23):
    rng = np.random.default_rng(seed)
    u = lambda shape, fan: rng.uniform(-1, 1, shape).astype(np.float32) / np.float32(np.sqrt(fan))
    return dict(f0=u((48, 5, 5, 1), 25), e1=u((64, 1, 1, 48), 48), g1=u((64, 3, 3, 8), 72), p1=u((48, 1, 1, 64), 64),
                e2=u((96, 1, 1, 48), 48), g2=u((96, 3, 3, 4), 36), p2=u((64, 1, 1, 96), 96), w8=u((10, 1, 1, 64), 64), b8=u(10, 64))


class ResNeXtLite:
    """stem conv 48@5x5 -> BN+ReLU (x0) -> [1x1 48->64, BN+ReLU, grouped 3x3/1 pad 1 G = 8 (Cg = 8), BN+ReLU, 1x1 64->48,
    BN + x0 with ReLU] (x1) -> [1x1 48->96, BN+ReLU, grouped 3x3/2 pad 1 G = 24 (Cg = 4, the narrow path), BN+ReLU, 1x1 96->64, BN]
    -> GAP -> fc 64->10 -> softmax CE (1/B).  The convs have no bias.  Every 1x1 conv reads >= 48 channels, so each is a
    wide-family layer, which has a 1x1 input gradient."""

    def __init__(self, eng, pkg, p):
        self.eng = eng
        relu, none = pkg.ACT_RELU, pkg.ACT_NONE
        B = NB
        conv = lambda H, C, K, R, f: pkg.ConvLayer(eng, B, H, H, C, K, R, R, p[f], None, act=none)
        self.stem = conv(28, 1, 48, 5, "f0")
        self.e1, self.p1 = conv(24, 48, 64, 1, "e1"), conv(24, 64, 48, 1, "p1")
        self.e2, self.p2 = conv(24, 48, 96, 1, "e2"), conv(12, 96, 64, 1, "p2")
        assert self.stem.family == "narrow" and all(c.family == "wide" for c in (self.e1, self.p1, self.e2, self.p2))
        self.g1 = pkg.GroupedConvLayer(eng, B, 24, 24, 64, 64, 8, 3, 3, p["g1"], None, act=none, stride=1, padding=(1, 1))
        self.g2 = pkg.GroupedConvLayer(eng, B, 24, 24, 96, 96, 24, 3, 3, p["g2"], None, act=none, stride=2, padding=(1, 1))
        assert self.g1.out_shape == (B, 24, 24, 64) and self.g2.out_shape == (B, 12, 12, 96)
        assert self.g1.info["vec"] == 8 and self.g2.info["vec"] == 4
        BN = lambda H, C, act: pkg.BatchNormLayer(eng, B, H, H, C, act=act)
        self.bn = [BN(24, 48, relu), BN(24, 64, relu), BN(24, 64, relu), BN(24, 48, relu), BN(24, 96, relu), BN(12, 96, relu),
                   BN(12, 64, none)]
        self.gap = pkg.GlobalAvgPoolLayer(eng, B, 12, 12, 64)
        self.fc = pkg.LinearLayer(eng, B, 1, 1, 64, 10, p["w8"], p["b8"], act=none, row_pitch=self.gap.row_pitch)
        buf = lambda *shape: torch.full(shape, NAN_BF16, dtype=torch.int16, device=DEV)
        self.y0, self.x0, self.dx0, self.dy0, self.dres, self.yp1, self.x1, self.dx1, self.dyp1 = (buf(B, 24, 24, 48) for _ in range(9))
        self.ye1, self.ze1, self.yg1, self.zg1, self.dzg1, self.dyg1, self.dze1, self.dye1 = (buf(B, 24, 24, 64) for _ in range(8))
        self.ye2, self.ze2, self.dze2, self.dye2 = (buf(B, 24, 24, 96) for _ in range(4))
        self.yg2, self.zg2, self.dzg2, self.dyg2 = (buf(B, 12, 12, 96) for _ in range(4))
        self.yp2, self.out, self.dout, self.dyp2 = (buf(B, 12, 12, 64) for _ in range(4))
        self.h, self.dh = buf(B, self.gap.row_pitch), buf(B, self.gap.row_pitch)
        self.z, self.dz = buf(B, 10), buf(B, 10)
        self.loss = torch.zeros(B, dtype=torch.float32, device=DEV)
        self.pred = torch.zeros(B, dtype=torch.int32, device=DEV)

    def forward(self, x, labels, training=True):
        b0, be1, bg1, bp1, be2, bg2, bp2 = self.bn
        self.stem.forward(x, self.y0)
        b0.forward(self.y0, self.x0, training=training)
        self.e1.forward(self.x0, self.ye1)
        be1.forward(self.ye1, self.ze1, training=training)
        self.g1.forward(self.ze1, self.yg1)
        bg1.forward(self.yg1, self.zg1, training=training)
        self.p1.forward(self.zg1, self.yp1)
        bp1.forward(self.yp1, self.x1, r=self.x0, training=training)
        self.e2.forward(self.x1, self.ye2)
        be2.forward(self.ye2, self.ze2, training=training)
        self.g2.forward(self.ze2, self.yg2)
        bg2.forward(self.yg2, self.zg2, training=training)
        self.p2.forward(self.zg2, self.yp2)
        bp2.forward(self.yp2, self.out, training=training)
        self.gap.forward(self.out, self.h)
        self.fc.forward(self.h, self.z)
        self.eng.softmax_ce_bf16(self.z, labels, NB, 10, 1.0 / NB, self.dz, self.loss, self.pred)

    def backward(self):
        b0, be1, bg1, bp1, be2, bg2, bp2 = self.bn
        self.fc.backward(self.z, self.dz, self.dh)
        self.gap.backward(self.dh, self.dout)
        bp2.backward(self.out, self.dout, self.dyp2)
        self.p2.backward(self.yp2, self.dyp2, self.dzg2)
        bg2.backward(self.zg2, self.dzg2, self.dyg2)
        self.g2.backward(self.yg2, self.dyg2, self.dze2)
        be2.backward(self.ze2, self.dze2, self.dye2)
        self.e2.backward(self.ye2, self.dye2, self.dx1)
        bp1.backward(self.x1, self.dx1, self.dyp1, dr=self.dres)
        self.p1.backward(self.yp1, self.dyp1, self.dzg1)
        bg1.backward(self.zg1, self.dzg1, self.dyg1)
        self.g1.backward(self.yg1, self.dyg1, self.dze1)
        be1.backward(self.ze1, self.dze1, self.dye1)
        self.e1.backward(self.ye1, self.dye1, self.dx0)
        b0.backward(self.x0, self.dx0, self.dy0, dy2=self.dres)                    # the block's two paths meet at x0
        self.stem.backward(self.y0, self.dy0, None)

    def layers(self):
        return (self.stem, self.e1, self.g1, self.p1, self.e2, self.g2, self.p2, self.fc, *self.bn)

    def sgd(self, lr):
        for layer in self.layers():
            layer.sgd(lr)

    def params(self):
        return [a for layer in self.layers() for a in layer.params() if a is not None]

    def close(self):
        for layer in (*self.layers(), self.gap):
            layer.close()


def mnist_device(pkg, u8):
    n = u8.shape[0]
    xl = np.zeros((n * 28, 32), np.uint16)
    xl[:, :28] = pkg.f32_to_bf16_bits(u8.reshape(n, 28, 28).astype(np.float32) / 255.0).reshape(n * 28, 28)
    return torch.from_numpy(xl.view(np.int16)).to(DEV)


def host(t):
    return t.cpu().numpy().view(np.uint16)


def test_resnext_mnist(eng, pkg, golden):
    """In each of the first 5 steps both grouped layers' y and dx are bit-exact against the replays on the device's own tensors
    and dw lies within its bound.  A fresh run reproduces the parameters after 5 steps bit for bit.  After EPOCHS epochs over the
    1024 training digits the mean loss has fallen, and test accuracy on the 256 test digits, evaluated with the running statistics,
    exceeds ACC_MIN."""
    xs, ys = mnist_device(pkg, golden["train_u8"]), torch.from_numpy(golden["train_labels"]).to(DEV)
    xt, yt = mnist_device(pkg, golden["test_u8"]), torch.from_numpy(golden["test_labels"]).to(DEV)
    row_bytes = 28 * 32 * 2
    batch = lambda s, xs=xs, ys=ys: (xs.data_ptr() + s * NB * row_bytes, ys[s * NB:(s + 1) * NB])

    net = ResNeXtLite(eng, pkg, init_params())
    for it in range(5):
        net.forward(*batch(it))
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
        net.sgd(LR_STEP)
        eng.sync()
    after5 = net.params()
    net.close()

    net = ResNeXtLite(eng, pkg, init_params())
    losses = []
    for ep in range(EPOCHS):
        for s in range(1024 // NB):
            net.forward(*batch(s))
            net.backward()
            net.sgd(LR_STEP)
            losses.append(net.loss)
            net.loss = torch.zeros(NB, dtype=torch.float32, device=DEV)
            if ep == 0 and s == 4:
                eng.sync()
                assert all(np.array_equal(a.view(np.uint32), b_.view(np.uint32)) for a, b_ in zip(net.params(), after5))
    eng.sync()
    ep_loss = [float(torch.stack(losses[e * 8:(e + 1) * 8]).double().mean()) for e in range(EPOCHS)]
    right = 0
    for s in range(2):
        net.forward(*batch(s, xt, yt), training=False)
        eng.sync()
        right += int((net.pred.cpu().numpy() == golden["test_labels"][s * NB:(s + 1) * NB]).sum())
    acc = right / 256
    net.close()
    print(f"ResNeXt-style network: mean loss by epoch {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}; test accuracy {acc:.4f} (threshold {ACC_MIN})")
    assert np.isfinite(ep_loss).all() and ep_loss[-1] < ep_loss[0]
    assert acc > ACC_MIN
