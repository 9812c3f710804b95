"""Batch normalization with a fused residual add and ReLU (pcnn_batchnorm_nhwc_bf16_fwd / _bwd, BatchNormLayer): y and dx bit for
bit against the float32 replays of batchnorm_ref.py on the device's own statistics and gradient sums, the statistics and the sums
within fp32 accumulation bounds of float64 (a large offset included), the whole BN + add + ReLU against torch autograd in float64,
buffers, reruns and refusals, one ConvLayer -> BatchNormLayer step, and a small ResNet-style network trained on MNIST digits.

Error model of the statistics (u = 2^-24).  Each CTA sums d = x - k and d * d in fp32, k one of the channel's own values, along
chains of at most ITERS (16) terms per thread and then `lanes` terms per CTA, and the CTA sums are merged in double.  With
R = max - min of the channel (so |d| <= R) and n = ITERS + lanes + 3:
    |mean - mean64| <= n u R + u |mean64|,      |var - var64| <= 5 n u R^2 + 4 u (var64 + eps)
(var read back from save_rstd as 1 / rstd^2 - eps, which adds the 4 u term).  The bound depends on the spread, not on the mean:
x = 4096 + 32 k keeps it tight where E[x^2] - E[x]^2 in fp32 is off by far more.  dbeta and dgamma sum in fp32 over ITERS terms
per thread, `lanes` per CTA and the CTAs in 8 interleaved chains added in a 3-level tree: n_acc = ITERS + lanes + ceil(ctas / 8)
+ 3 additions, so |s - s64| <= 2 (n_acc + 1) u sum |term|."""
import numpy as np
import pytest
import torch

import batchnorm_ref as BR
import conv_ref as CR
import conv_ref_strided as CS
from batchnorm_ref import ITERS, U, check_stats, n_acc, n_stat  # noqa: F401
from example_nets import NAN_BF16, ResNet, host, train

pytestmark = pytest.mark.gpu

TAIL = 64

CS_ = [1, 6, 8, 16, 64, 120, 256]
PIXELS = [2, 7, 1001]
GRID = [(C, p) for C in CS_ for p in PIXELS] + [(64, 128 * 56 * 56)]
GIDS = [f"C{C}-px{p}" for C, p in GRID]


def bits(pkg, a):
    return pkg.f32_to_bf16_bits(np.asarray(a, np.float32))


class Stats:
    """gamma, beta, running and saved statistics of one call, fp32 [C] DeviceArrays"""

    def __init__(self, eng, gamma, beta, rm, rv):
        C = gamma.size
        self.gamma, self.beta = eng.to_device(np.asarray(gamma, np.float32)), eng.to_device(np.asarray(beta, np.float32))
        self.rm, self.rv = eng.to_device(np.asarray(rm, np.float32)), eng.to_device(np.asarray(rv, np.float32))
        self.sm, self.sr = eng.to_device(np.full(C, np.nan, np.float32)), eng.to_device(np.full(C, np.nan, np.float32))

    def free(self):
        for a in (self.gamma, self.beta, self.rm, self.rv, self.sm, self.sr):
            a.free()


def operands(pkg, rng, pixels, C, offset=None):
    x = rng.standard_normal((pixels, C)) * rng.uniform(0.5, 2, C) + (rng.uniform(-4, 4, C) if offset is None else offset)
    gamma, beta = rng.uniform(0.5, 1.5, C), rng.uniform(-0.5, 0.5, C)
    r = rng.standard_normal((pixels, C))
    rm, rv = rng.uniform(-1, 1, C), rng.uniform(0.5, 2, C)
    return bits(pkg, x), bits(pkg, r), gamma.astype(np.float32), beta.astype(np.float32), rm.astype(np.float32), rv.astype(np.float32)


def run_fwd(eng, xb, rb, st, act, training, eps=1e-5, momentum=0.1):
    pixels, C = xb.shape
    xd = eng.to_device(xb)
    rd = None if rb is None else eng.to_device(rb)
    y = eng.to_device(np.full(pixels * C + TAIL, NAN_BF16, np.uint16))
    eng.batchnorm_fwd(xd, y, pixels, C, st.gamma, st.beta, st.rm, st.rv, st.sm, st.sr, r=rd, act=act, training=training, eps=eps,
                      momentum=momentum)
    eng.sync()
    out = y.to_host()
    for a in (xd, rd, y):
        if a is not None:
            a.free()
    return out


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("C,pixels", GRID, ids=GIDS)
def test_forward(eng, pkg, C, pixels):
    """training and eval, act 0 and 3, with and without r: y bit-identical to the replay (from save_mean / save_rstd, or from the
    running statistics in eval), NaN-prefilled y fully written and its tail untouched, statistics within the error model,
    running_mean bit-identical to its replay and running_var within bound, reruns bit-identical"""
    rng = np.random.default_rng(C * 1009 + pixels)
    xb, rb, gamma, beta, rm0, rv0 = operands(pkg, rng, pixels, C)
    n = pixels * C
    big = pixels > 10000
    combos = [(a, wr) for a in (0, 3) for wr in (False, True)] if not big else [(3, True), (0, False)]
    for act, with_r in combos:
        r = rb if with_r else None
        for training in (True, False):
            st = Stats(eng, gamma, beta, rm0, rv0)
            y = run_fwd(eng, xb, r, st, act, training)
            assert np.all(y[n:] == NAN_BF16)
            if training:
                mean, rstd = st.sm.to_host(), st.sr.to_host()
                _, v64, vb = check_stats(pkg, xb, mean, rstd, 1e-5)
                assert np.array_equal(st.rm.to_host(), BR.running_update(rm0, mean, 0.1))
                unbiased = v64 * pixels / (pixels - 1)
                want_rv = 0.9 * rv0.astype(np.float64) + 0.1 * unbiased
                assert np.all(np.abs(st.rv.to_host() - want_rv) <= 0.1 * vb * pixels / (pixels - 1) + 4 * U * np.abs(want_rv))
            else:
                mean, rstd = rm0, BR.eval_rstd(rv0, 1e-5)
                assert np.array_equal(st.rm.to_host(), rm0) and np.array_equal(st.rv.to_host(), rv0)
                assert np.all(np.isnan(st.sm.to_host()))                  # eval writes no saved statistics
            want = BR.fwd_bits(pkg, xb, gamma, beta, mean, rstd, r, act)
            assert np.array_equal(y[:n].reshape(pixels, C), want), (act, with_r, training)
            if act == 3 and with_r:                                      # a rerun: same y, same saved statistics
                again = run_fwd(eng, xb, r, st, act, training)
                assert np.array_equal(again, y) and (not training or np.array_equal(st.sm.to_host(), mean))
            st.free()


@pytest.mark.parametrize("C,pixels", [(C, p) for C in CS_ for p in (2, 1000)] + [(64, 128 * 56 * 56)])
def test_forward_near_exact(eng, pkg, C, pixels):
    """eps = 0 and each channel holds m +- 2^k in equal numbers: save_mean within 1 ulp of m and save_rstd within 1 ulp of 2^-k"""
    rng = np.random.default_rng(C + pixels)
    k = rng.integers(-3, 4, C)
    m = rng.integers(-20, 21, C) * 2.0 ** (k + 2)
    sign = np.where(rng.permuted(np.tile(np.arange(pixels) % 2, (C, 1)), axis=1).T == 0, 1.0, -1.0)
    x = m + sign * 2.0 ** k
    xb = bits(pkg, x)
    assert np.array_equal(pkg.bf16_bits_to_f32(xb), x.astype(np.float32))
    st = Stats(eng, np.ones(C), np.zeros(C), np.zeros(C), np.ones(C))
    run_fwd(eng, xb, None, st, 0, True, eps=0.0)
    mean, rstd = st.sm.to_host(), st.sr.to_host()
    ulp = lambda v: np.spacing(np.abs(np.float32(v)).astype(np.float32))
    assert np.all(np.abs(mean - m) <= np.maximum(ulp(m), np.float32(2.0 ** -149)))
    assert np.all(np.abs(rstd - 2.0 ** -k) <= ulp(2.0 ** -k))
    st.free()


@pytest.mark.parametrize("C,pixels", [(1, 1001), (8, 1001), (64, 1001), (120, 1001), (64, 128 * 56 * 56)])
def test_forward_offset(eng, pkg, C, pixels):
    """x = 4096 + 32 k, k in -3..3 (the bf16 grid at 4096 is 32 apart): the variance error stays within the model, which naive
    E[x^2] - E[x]^2 summed in fp32 breaks"""
    rng = np.random.default_rng(C)
    x = 4096.0 + 32.0 * rng.integers(-3, 4, (pixels, C))
    xb = bits(pkg, x)
    assert np.array_equal(pkg.bf16_bits_to_f32(xb), x.astype(np.float32))
    st = Stats(eng, np.ones(C), np.zeros(C), np.zeros(C), np.ones(C))
    run_fwd(eng, xb, None, st, 0, True)
    _, v64, bound = check_stats(pkg, xb, st.sm.to_host(), st.sr.to_host(), 1e-5)
    assert np.all(bound <= 1e-3 * v64)
    x32 = x.astype(np.float32)
    naive = np.cumsum(x32 * x32, axis=0, dtype=np.float32)[-1] / np.float32(pixels) - (np.cumsum(x32, axis=0, dtype=np.float32)[-1] / np.float32(pixels)) ** 2
    if pixels * C >= 64 * 1001:                                         # enough terms for the naive sum to go wrong
        assert np.any(np.abs(naive - v64) > bound)
    st.free()


# ------------------------------------------------------------------------------------------------ backward
def run_bwd(eng, xb, yb, dyb, st, act, dy2b=None, with_dr=True, in_place=False):
    pixels, C = xb.shape
    n = pixels * C
    xd, yd = eng.to_device(xb), eng.to_device(yb)
    dyd = eng.to_device(np.concatenate([dyb.reshape(-1), np.full(TAIL, NAN_BF16, np.uint16)]))
    dy2d = None if dy2b is None else eng.to_device(dy2b)
    dx = dyd if in_place else eng.to_device(np.full(n + TAIL, NAN_BF16, np.uint16))
    dr = eng.to_device(np.full(n + TAIL, NAN_BF16, np.uint16)) if with_dr else None
    dg, db = eng.to_device(np.full(C, np.nan, np.float32)), eng.to_device(np.full(C, np.nan, np.float32))
    eng.batchnorm_bwd(xd, yd, dyd, st.gamma, st.sm, st.sr, dx, dg, db, pixels, C, act=act, dy2=dy2d, dr=dr)
    eng.sync()
    out = dx.to_host(), (dr.to_host() if with_dr else None), dg.to_host(), db.to_host()
    for a in {id(v): v for v in (xd, yd, dyd, dy2d, dx, dr, dg, db) if v is not None}.values():
        a.free()
    return out


@pytest.mark.parametrize("C,pixels", GRID, ids=GIDS)
def test_backward(eng, pkg, C, pixels):
    """act 0 and 3, with and without dy2: dr bit-identical to g~, dbeta and dgamma within the fp32 bound of float64, dx
    bit-identical to the replay from the device's dgamma, dbeta and statistics, NaN-prefilled outputs fully written with tails
    untouched; dy2 equals the backward of the pre-added dy; in place equals out of place; reruns bit-identical"""
    rng = np.random.default_rng(C * 31 + pixels)
    xb, rb, gamma, beta, rm0, rv0 = operands(pkg, rng, pixels, C)
    n = pixels * C
    f32 = pkg.bf16_bits_to_f32
    big = pixels > 10000
    for act in (0, 3):
        st = Stats(eng, gamma, beta, rm0, rv0)
        yb = run_fwd(eng, xb, rb, st, act, True)[:n].reshape(pixels, C)
        mean, rstd = st.sm.to_host(), st.sr.to_host()
        dyb = bits(pkg, rng.standard_normal((pixels, C)))
        dy2b = bits(pkg, rng.standard_normal((pixels, C)))
        for d2 in ((None, dy2b) if not big or act == 3 else (None,)):
            dx, dr, dg, db = run_bwd(eng, xb, yb, dyb, st, act, d2)
            assert np.all(dx[n:] == NAN_BF16) and np.all(dr[n:] == NAN_BF16)
            g = BR.grad_bits(pkg, yb, dyb, d2, act)
            assert np.array_equal(dr[:n].reshape(pixels, C), g)
            gf = f32(g).astype(np.float64)
            xh = BR.xhat32(pkg, xb, mean, rstd).astype(np.float64)
            na = n_acc(pkg, pixels, C)
            assert np.all(np.abs(db - gf.sum(0)) <= 2 * (na + 1) * U * np.abs(gf).sum(0))
            assert np.all(np.abs(dg - (gf * xh).sum(0)) <= 2 * (na + 1) * U * np.abs(gf * xh).sum(0))
            want = BR.dx_bits(pkg, xb, g, gamma, mean, rstd, dg, db)
            assert np.array_equal(dx[:n].reshape(pixels, C), want), (act, d2 is None)
            if d2 is not None:                                           # dy2 = the backward of the pre-added dy
                pre = run_bwd(eng, xb, yb, pkg.f32_to_bf16_bits(f32(dyb) + f32(d2)), st, act)
                assert all(np.array_equal(a.view(np.uint16 if a.dtype == np.uint16 else np.uint32),
                                          b.view(np.uint16 if b.dtype == np.uint16 else np.uint32))
                           for a, b in zip((dx, dr, dg, db), pre))
            else:
                ip = run_bwd(eng, xb, yb, dyb, st, act, None, with_dr=False, in_place=True)
                assert np.array_equal(ip[0], dx) and np.array_equal(ip[2].view(np.uint32), dg.view(np.uint32))
                again = run_bwd(eng, xb, yb, dyb, st, act, None)
                assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(again, (dx, dr, dg, db)))
        st.free()


@pytest.mark.parametrize("C,pixels", [(6, 1001), (64, 1001), (64, 128 * 56 * 56)])
def test_backward_integer_dbeta_exact(eng, pkg, C, pixels):
    """dy in -2..2 at act 3: every partial sum of dbeta is an integer below 2^24, so dbeta equals the float64 sum bit for bit"""
    rng = np.random.default_rng(C + 17)
    xb, rb, gamma, beta, rm0, rv0 = operands(pkg, rng, pixels, C)
    st = Stats(eng, gamma, beta, rm0, rv0)
    yb = run_fwd(eng, xb, rb, st, 3, True)[:pixels * C].reshape(pixels, C)
    dyb = bits(pkg, rng.integers(-2, 3, (pixels, C)))
    _, _, _, db = run_bwd(eng, xb, yb, dyb, st, 3, None, with_dr=False)
    g = pkg.bf16_bits_to_f32(BR.grad_bits(pkg, yb, dyb, None, 3)).astype(np.float64)
    assert np.array_equal(db.astype(np.float64), g.sum(0))
    st.free()


@pytest.mark.parametrize("act,with_r,with_dy2", [(3, True, True), (3, False, False), (0, True, False), (0, False, True)])
def test_against_torch_autograd(eng, pkg, act, with_r, with_dy2):
    """BN + add + ReLU on bf16-rounded inputs, against torch autograd in float64: y within bf16 rounding, dx within a bf16-sized
    bound of the terms it is made of, dgamma and dbeta within 2^-7 of their magnitude"""
    N, H, W, C = 4, 5, 7, 16
    M = N * H * W
    rng = np.random.default_rng(act + 2 * with_r + 4 * with_dy2)
    f32 = pkg.bf16_bits_to_f32
    xb, rb, gamma, beta, rm0, rv0 = operands(pkg, rng, M, C)
    r = rb if with_r else None
    dyb, dy2b = bits(pkg, rng.standard_normal((M, C))), (bits(pkg, rng.standard_normal((M, C))) if with_dy2 else None)
    st = Stats(eng, gamma, beta, rm0, rv0)
    yb = run_fwd(eng, xb, r, st, act, True)[:M * C].reshape(M, C)
    dx, dr, dg, db = run_bwd(eng, xb, yb, dyb, st, act, dy2b)
    xt = torch.from_numpy(f32(xb).astype(np.float64)).reshape(N, H, W, C).permute(0, 3, 1, 2).requires_grad_(True)
    gt = torch.from_numpy(gamma.astype(np.float64)).requires_grad_(True)
    bt = torch.from_numpy(beta.astype(np.float64)).requires_grad_(True)
    v = torch.nn.functional.batch_norm(xt, None, None, gt, bt, training=True, eps=1e-5)
    if r is not None:
        v = v + torch.from_numpy(f32(r).astype(np.float64)).reshape(N, H, W, C).permute(0, 3, 1, 2)
    if act == 3:
        v = torch.relu(v)
    y64 = v.detach().permute(0, 2, 3, 1).reshape(M, C).numpy()
    assert np.all(np.abs(f32(yb) - y64) <= 2.0 ** -8 * np.abs(y64) + 1e-5)
    t = f32(dyb).astype(np.float64) + (0 if dy2b is None else f32(dy2b).astype(np.float64))
    v.backward(torch.from_numpy(t).reshape(N, H, W, C).permute(0, 3, 1, 2))
    dx64 = xt.grad.permute(0, 2, 3, 1).reshape(M, C).numpy()
    x64 = f32(xb).astype(np.float64)
    rstd64 = 1 / np.sqrt(x64.var(0) + 1e-5)
    xh = (x64 - x64.mean(0)) * rstd64
    gabs = np.abs(t)
    scale = np.abs(gamma * rstd64) * (gabs + np.abs(bt.grad.numpy()) / M + np.abs(xh) * np.abs(gt.grad.numpy()) / M)
    assert np.all(np.abs(f32(dx[:M * C]).reshape(M, C) - dx64) <= 2.0 ** -6 * scale + 1e-6)
    assert np.all(np.abs(dg - gt.grad.numpy()) <= 2.0 ** -7 * np.abs(gabs * xh).sum(0))
    assert np.all(np.abs(db - bt.grad.numpy()) <= 2.0 ** -7 * gabs.sum(0))
    st.free()


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(eng, pkg):
    pixels, C = 64, 16
    n = pixels * C
    t = [eng.array(n + 64, np.uint16) for _ in range(6)]
    x, r, y, dy, dx, dr = t
    v = [eng.array(C + 8) for _ in range(8)]
    gamma, beta, rm, rv, sm, sr, dg, db = v
    fwd = lambda **kw: eng.batchnorm_fwd(**{**dict(x=x, y=y, pixels=pixels, C=C, gamma=gamma, beta=beta, running_mean=rm, running_var=rv,
                                                   save_mean=sm, save_rstd=sr, r=r, act=3, training=True, eps=1e-5, momentum=0.1), **kw})
    bwd = lambda **kw: eng.batchnorm_bwd(**{**dict(x=x, y=y, dy=dy, gamma=gamma, save_mean=sm, save_rstd=sr, dx=dx, dgamma=dg, dbeta=db,
                                                   pixels=pixels, C=C, act=3, dy2=None, dr=dr), **kw})
    F, B = "pcnn_batchnorm_nhwc_bf16_fwd", "pcnn_batchnorm_nhwc_bf16_bwd"
    esc = lambda s: s.replace("(", r"\(").replace(")", r"\)").replace("*", r"\*").replace("+", r"\+")
    cases = [
        (lambda: fwd(act=1), F + ": act 1 (sigmoid) is not available after batch normalization: sigmoid_bf16 uses tanh.approx"),
        (lambda: bwd(act=1), B + ": act 1 (sigmoid) is not available"),
        (lambda: fwd(act=2), F + ": act 2 is not 0 (none) or 3 (ReLU)"),
        (lambda: bwd(act=-1), B + ": act -1 is not 0 (none) or 3 (ReLU)"),
        (lambda: fwd(C=0), F + ": C = 0 channels: 1 <= C <= 256 is required"),
        (lambda: fwd(C=257), "1 <= C <= 256 is required"),
        (lambda: bwd(C=300), B + ": C = 300 channels"),
        (lambda: fwd(pixels=1), "pixels = 1: training needs more than 1 value per channel"),
        (lambda: bwd(pixels=1), B + ": pixels = 1: training needs more than 1 value per channel"),
        (lambda: fwd(pixels=0, training=False), "pixels = 0: at least one pixel"),
        (lambda: fwd(eps=-1.0), "eps = -1: a finite eps >= 0 is required"),
        (lambda: fwd(eps=float("inf")), "a finite eps >= 0 is required"),
        (lambda: fwd(eps=float("nan")), "a finite eps >= 0 is required"),
        (lambda: fwd(momentum=1.5), "momentum = 1.5: 0 <= momentum <= 1 is required"),
        (lambda: fwd(momentum=-0.1), "0 <= momentum <= 1 is required"),
        (lambda: fwd(momentum=float("nan")), "0 <= momentum <= 1 is required"),
        (lambda: fwd(x=None), F + ": NULL context, x, y, gamma or beta"),
        (lambda: fwd(y=None), "NULL context, x, y, gamma or beta"),
        (lambda: fwd(gamma=None), "NULL context, x, y, gamma or beta"),
        (lambda: fwd(beta=None), "NULL context, x, y, gamma or beta"),
        (lambda: fwd(save_mean=None), "training needs save_mean and save_rstd"),
        (lambda: fwd(save_rstd=None), "training needs save_mean and save_rstd"),
        (lambda: fwd(running_var=None), "running_mean and running_var must both be given or both be NULL"),
        (lambda: fwd(running_mean=None, training=False), "eval (training = 0) needs running_mean and running_var"),
        (lambda: bwd(dy=None), B + ": NULL context, x, y, dy, gamma, save_mean, save_rstd, dx, dgamma or dbeta"),
        (lambda: bwd(x=None), "NULL context, x, y, dy"),
        (lambda: bwd(y=None), "NULL context, x, y, dy"),
        (lambda: bwd(dx=None), "NULL context, x, y, dy"),
        (lambda: bwd(dgamma=None), "NULL context, x, y, dy"),
        (lambda: bwd(save_rstd=None), "NULL context, x, y, dy"),
        (lambda: fwd(x=x.ptr + 2), "must be 16-byte aligned"),
        (lambda: fwd(r=r.ptr + 8), "must be 16-byte aligned"),
        (lambda: fwd(gamma=gamma.ptr + 4), "must be 16-byte aligned"),
        (lambda: bwd(dy2=dr.ptr + 2), "must be 16-byte aligned"),
        (lambda: bwd(dbeta=db.ptr + 4), "must be 16-byte aligned"),
        (lambda: fwd(y=x), F + ": overlapping buffers"),
        (lambda: fwd(r=y), "overlapping buffers"),
        (lambda: fwd(y=x.ptr + 16), "overlapping buffers"),
        (lambda: fwd(save_mean=rm), "overlapping buffers"),
        (lambda: fwd(beta=gamma), "overlapping buffers"),
        (lambda: bwd(dx=dy.ptr + 16), B + ": overlapping buffers: only dx == dy (in place) may share memory"),
        (lambda: bwd(dx=x), "only dx == dy (in place) may share memory"),
        (lambda: bwd(dr=dy), "only dx == dy (in place) may share memory"),
        (lambda: bwd(dr=dx), "only dx == dy (in place) may share memory"),
        (lambda: bwd(dgamma=db), "only dx == dy (in place) may share memory"),
    ]
    for fn, msg in cases:
        with pytest.raises(pkg.PcnnError, match=esc(msg)):
            fn()
    fwd(r=None, running_mean=None, running_var=None)                    # training without running statistics is allowed
    fwd(training=False, save_mean=None, save_rstd=None)
    bwd(dx=dy, dr=None)                                                  # in place
    eng.sync()
    for a in t + v:
        a.free()



# ------------------------------------------------------------------------------------------------ layer step
def test_conv_bn_relu_step(eng, pkg):
    """ConvLayer (no bias) -> BatchNormLayer (ReLU), one step: the conv y within the bound of test_conv_train_gpu.py, the BN y and
    dx bit-exact against the replays on the device's tensors, the conv gradients against float64 on the device's BN dx, and
    every sgd update bit-identical to w + (-lr) * dw in numpy float32"""
    N, H, W, C, K, R, S, pad = 4, 12, 12, 8, 16, 3, 3, 1
    P, Q = H, W
    rng = np.random.default_rng(21)
    f32 = pkg.bf16_bits_to_f32
    x = f32(bits(pkg, rng.uniform(0, 1, (N, H, W, C))))
    f = f32(bits(pkg, rng.uniform(-0.5, 0.5, (K, R, S, C))))
    gamma, beta = rng.uniform(0.5, 1.5, K).astype(np.float32), rng.uniform(-0.5, 0.5, K).astype(np.float32)
    conv = pkg.ConvLayer(eng, N, H, W, C, K, R, S, f, None, act=pkg.ACT_NONE, padding=(pad, pad))
    bn = pkg.BatchNormLayer(eng, N, P, Q, K, act=pkg.ACT_RELU, gamma=gamma, beta=beta)
    pitch = conv.row_pitch
    xl = np.zeros((N * H, pitch), np.uint16)
    xl[:, :W * C] = bits(pkg, x).reshape(N * H, W * C)
    xd = eng.to_device(xl)
    yc, z = eng.to_device(np.full((N, P, Q, K), NAN_BF16, np.uint16)), eng.to_device(np.full((N, P, Q, K), NAN_BF16, np.uint16))
    dz = eng.to_device(bits(pkg, rng.standard_normal((N, P, Q, K))))
    dyc = eng.to_device(np.full((N, P, Q, K), NAN_BF16, np.uint16))
    dx = eng.to_device(np.full((N * H, pitch), NAN_BF16, np.uint16))
    conv.forward(xd, yc)
    bn.forward(yc, z)
    bn.backward(z, dz, dyc)
    conv.backward(yc, dyc, dx)
    eng.sync()
    M = N * P * Q
    ycb, zb, dzb, dycb = (a.to_host().reshape(M, K) for a in (yc, z, dz, dyc))
    xp = np.pad(x.astype(np.float64), ((0, 0), (pad, pad), (pad, pad), (0, 0)))
    pre = CR.conv_fwd_f64(xp, f, np.zeros(K), 1)
    pre_abs = CR.conv_fwd_f64(np.abs(xp), np.abs(f), np.zeros(K), 1)
    assert np.all(np.abs(f32(ycb).reshape(N, P, Q, K) - pre) <= 2 * R * S * C * U * pre_abs + 2.0 ** -8 * np.abs(pre))
    mean, rstd = bn.save_mean.to_host(), bn.save_rstd.to_host()
    check_stats(pkg, ycb, mean, rstd, 1e-5)
    assert np.array_equal(zb, BR.fwd_bits(pkg, ycb, gamma, beta, mean, rstd, None, 3))
    assert 0.2 < float((f32(zb) > 0).mean()) < 0.8
    g = BR.grad_bits(pkg, zb, dzb, None, 3)
    dg, db = bn.dgamma.to_host(), bn.dbeta.to_host()
    assert np.array_equal(dycb, BR.dx_bits(pkg, ycb, g, gamma, mean, rstd, dg, db))
    d = f32(dycb).astype(np.float64).reshape(N, P, Q, K)
    dw = CS.conv_wgrad_f64(xp, d, R, S, 1)
    dw_abs = CS.conv_wgrad_f64(np.abs(xp), np.abs(d), R, S, 1)
    assert np.all(np.abs(conv.dw.to_host() - dw) <= 2 * M * U * dw_abs + 1e-30)
    dx_ref = CS.conv_dgrad_f64(d, f.astype(np.float64), H + 2 * pad, W + 2 * pad, 1)[:, pad:pad + H, pad:pad + W, :]
    dx_abs = CS.conv_dgrad_f64(np.abs(d), np.abs(f.astype(np.float64)), H + 2 * pad, W + 2 * pad, 1)[:, pad:pad + H, pad:pad + W, :]
    got_dx = f32(dx.to_host()[:, :W * C].reshape(N, H, W, C)).astype(np.float64)
    assert np.all(np.abs(got_dx - dx_ref) <= 2.0 ** -8 * np.abs(dx_ref) + 2 * K * R * S * U * dx_abs + 1e-30)
    lr = np.float32(0.05)
    w0, g0, b0 = conv.params()[0], bn.gamma.to_host(), bn.beta.to_host()
    dw_dev = conv.dw.to_host()
    conv.sgd(float(lr))
    bn.sgd(float(lr))
    eng.sync()
    assert np.array_equal(conv.params()[0], w0 + (-lr) * dw_dev)
    g1, b1, rm1, rv1 = bn.params()
    assert np.array_equal(g1, g0 + (-lr) * dg) and np.array_equal(b1, b0 + (-lr) * db)
    assert np.array_equal(rm1, BR.running_update(np.zeros(K, np.float32), mean, 0.1))
    for a in (xd, yc, z, dz, dyc, dx):
        a.free()
    conv.close()
    bn.close()


# ------------------------------------------------------------------------------------------------ end to end
ACC_MIN = 0.90          # a float32 torch CPU replica of this network, initialisation and step reaches 0.973


def test_resnet_mnist(eng, pkg, golden):
    """In each of the first 5 steps every BN's y and dx are bit-exact against the replays on the device's own x, r, dy, dy2,
    statistics and gradient sums.  A second fresh run reproduces the parameters after 5 steps bit for bit.  After EPOCHS epochs
    over the 1024 training digits the mean loss has fallen, and test accuracy on the 256 test digits, evaluated with the running
    statistics, exceeds ACC_MIN."""

    def check_step(net, it, x, labels):
        net.forward(x, labels)
        eng.sync()
        fwd = [(bn, host(x), None if r is None else host(r), host(y), bn.save_mean.to_host(), bn.save_rstd.to_host(), bn.params())
               for bn, x, r, y, _, _, _ in net.bn_tensors()]
        net.backward()
        eng.sync()
        for (bn, xb, rb, yb, mean, rstd, (g, b, _, _)), (_, _, _, _, dy, dy2, dx) in zip(fwd, net.bn_tensors()):
            C = bn.shape[3]
            xb, yb = xb.reshape(-1, C), yb.reshape(-1, C)
            assert np.array_equal(yb, BR.fwd_bits(pkg, xb, g, b, mean, rstd, None if rb is None else rb.reshape(-1, C), 3)), it
            gt = BR.grad_bits(pkg, yb, host(dy).reshape(-1, C), None if dy2 is None else host(dy2).reshape(-1, C), 3)
            want = BR.dx_bits(pkg, xb, gt, g, mean, rstd, bn.dgamma.to_host(), bn.dbeta.to_host())
            assert np.array_equal(host(dx).reshape(-1, C), want), it
            frac = float((pkg.bf16_bits_to_f32(yb) > 0).mean())
            assert 0.1 < frac < 0.95, (it, frac)        # the ReLU is neither dead nor linear

    ep_loss, acc, _ = train(eng, pkg, golden, lambda: ResNet(eng, pkg, ResNet.init_params()), ResNet.EPOCHS, check_step=check_step)
    print(f"BN ResNet: mean loss by epoch {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}; test accuracy {acc:.4f} (threshold {ACC_MIN})")
    assert np.isfinite(ep_loss).all() and ep_loss[-1] < ep_loss[0]
    assert acc > ACC_MIN
