"""Group normalization on the device (pcnn_groupnorm_nhwc_bf16_fwd / _bwd / _bwd_preact): y, g (= dr) and dx bit for bit
against the float32 replays of groupnorm_ref.py on the device's own statistics and group sums (dstat), with every activation
code, r, dy2 and special values; the statistics, dgamma, dbeta and dstat within the error model of float64; each image alone
bit-identical to the same image anywhere in a batch of 128; buffers, in-place calls, reruns and refusals; and a GroupNormLayer
step under SGD and AdamW against optim_ref's replays.

The shapes are a covering set: Cg in {1, 2, 4, 8, 16, 32, C} (groups narrower than, as wide as and wider than a 16-byte vector,
and groups across a channel slice), C in {1, 3, 6, 8, 16, 64, 256, 320, 2048}, HW in {1, 7, 49, 784, 3136}, N in {1, 2, 3, 128},
and the four shapes scripts/conv_bench.py gn times, at their sizes."""
import numpy as np
import pytest

import bnact_ref as BA
import groupnorm_ref as GR
import optim_ref as OR
from example_nets import NAN_BF16

pytestmark = pytest.mark.gpu

TAIL = 64
SMS = 132
ACTS = [0, 3, 4, 5, 6]


def bits(pkg, a):
    return pkg.f32_to_bf16_bits(np.asarray(a, np.float32))


def same_or_nan(got, want):
    """bf16 bits: identical where want is a number; NaN (any payload) where want is NaN"""
    got, want = np.asarray(got, np.uint16), np.asarray(want, np.uint16)
    nan, gnan = (want & 0x7FFF) > 0x7F80, (got & 0x7FFF) > 0x7F80
    return np.array_equal(gnan, nan) and np.array_equal(got[~nan], want[~nan])


def nan_bf16(n):
    return np.full(n + TAIL, NAN_BF16, np.uint16)


def operands(pkg, rng, N, HW, C):
    """x with a mean and spread per channel, gamma in (0.5, 4) and beta in (-4, 7) so that v crosses every activation's knees, r
    and the incoming gradients wide"""
    x = rng.standard_normal((N, HW, C)) * rng.uniform(0.5, 2, C) + rng.uniform(-4, 4, C)
    gamma, beta = rng.uniform(0.5, 4, C).astype(np.float32), rng.uniform(-4, 7, C).astype(np.float32)
    r = rng.standard_normal((N, HW, C)) * 4
    dy, dy2 = rng.standard_normal((N, HW, C)), rng.standard_normal((N, HW, C))
    return bits(pkg, x), bits(pkg, r), gamma, beta, bits(pkg, dy), bits(pkg, dy2)


class Run:
    """one forward and one backward on the device, every output NaN-prefilled with a tail of TAIL elements past it"""

    def __init__(self, eng, pkg, xb, gamma, beta, G, act, rb=None, eps=1e-5):
        self.eng, self.pkg, self.G, self.act, self.eps = eng, pkg, G, act, eps
        self.N, self.HW, self.C = xb.shape
        self.xb, self.rb, self.gamma, self.beta = xb, rb, gamma, beta
        self.xd = eng.to_device(xb)
        self.rd = None if rb is None else eng.to_device(rb)
        self.gd, self.bd = eng.to_device(gamma), eng.to_device(beta)
        NG = self.N * G
        self.md, self.sd = eng.to_device(np.full(NG + TAIL, np.nan, np.float32)), eng.to_device(np.full(NG + TAIL, np.nan, np.float32))
        self.yd = eng.to_device(nan_bf16(xb.size))
        self.owned = [self.xd, self.rd, self.gd, self.bd, self.md, self.sd, self.yd]

    def fwd(self):
        self.eng.groupnorm_fwd(self.xd, self.yd, self.N, self.HW, self.C, self.G, self.gd, self.bd, self.md, self.sd, r=self.rd, act=self.act,
                               eps=self.eps)
        self.eng.sync()
        y, m, s = self.yd.to_host(), self.md.to_host(), self.sd.to_host()
        NG = self.N * self.G
        assert np.all(y[self.xb.size:] == NAN_BF16) and np.all(np.isnan(m[NG:])) and np.all(np.isnan(s[NG:]))
        self.y = y[:self.xb.size].reshape(self.xb.shape)
        self.mean, self.rstd = m[:NG].reshape(self.N, self.G), s[:NG].reshape(self.N, self.G)
        return self.y, self.mean, self.rstd

    def bwd(self, dyb, dy2b=None, with_dr=True, in_place=False):
        eng, n, C, NG = self.eng, self.xb.size, self.C, self.N * self.G
        dyd = eng.to_device(np.concatenate([dyb.reshape(-1), nan_bf16(0)]))
        dy2d = None if dy2b is None else eng.to_device(dy2b)
        dx = dyd if in_place else eng.to_device(nan_bf16(n))
        dr = eng.to_device(nan_bf16(n)) if with_dr else None
        dg, db = eng.to_device(np.full(C + TAIL, np.nan, np.float32)), eng.to_device(np.full(C + TAIL, np.nan, np.float32))
        ds = eng.to_device(np.full(2 * NG + TAIL, np.nan, np.float32))
        if self.act in BA.CODES:
            eng.groupnorm_bwd_preact(self.xd, dyd, self.gd, self.bd, self.md, self.sd, dx, dg, db, ds, self.N, self.HW, C, self.G, self.act,
                                     r=self.rd, dy2=dy2d, dr=dr)
        else:
            eng.groupnorm_bwd(self.xd, self.yd, dyd, self.gd, self.md, self.sd, dx, dg, db, ds, self.N, self.HW, C, self.G, act=self.act,
                              dy2=dy2d, dr=dr)
        eng.sync()
        out = [a.to_host() if a is not None else None for a in (dx, dr, dg, db, ds)]
        for a in {id(v): v for v in (dyd, dy2d, dx, dr, dg, db, ds) if v is not None}.values():
            a.free()
        for a, m in zip(out, (n, n, C, C, 2 * NG)):       # the TAIL elements past each output are untouched
            if a is not None:
                assert np.all(a[m:] == NAN_BF16) if a.dtype == np.uint16 else np.all(np.isnan(a[m:]))
        dxh = out[0][:n].reshape(self.xb.shape)
        drh = None if out[1] is None else out[1][:n].reshape(self.xb.shape)
        return dxh, drh, out[2][:C], out[3][:C], out[4][:2 * NG].reshape(2, self.N, self.G)

    def free(self):
        for a in self.owned:
            if a is not None:
                a.free()


def check_all(eng, pkg, xb, rb, gamma, beta, dyb, dy2b, G, act, stats=True):
    """forward and backward at act: y, g = dr and dx bit-exact against the replays on the device's statistics and dstat, the
    statistics and the sums within their bounds; returns the outputs and the worst ratios to the bounds"""
    N, HW, C = xb.shape
    info = pkg.groupnorm_nhwc_info(N, HW, C, G)
    run = Run(eng, pkg, xb, gamma, beta, G, act, rb)
    try:
        y, mean, rstd = run.fwd()
        assert same_or_nan(y, GR.fwd_bits(pkg, xb, gamma, beta, mean, rstd, rb, act)), ("y", act)
        if stats:
            GR.check_stats(pkg, xb, G, mean, rstd, 1e-5, info["n_acc_group"])
        dx, dr, dg, db, ds = run.bwd(dyb, dy2b)
        g = GR.grad_bits(pkg, xb, gamma, beta, mean, rstd, dyb, dy2b, rb if act in BA.CODES else None, act, y)
        assert same_or_nan(dr, g), ("dr", act)
        assert same_or_nan(dx, GR.dx_bits(pkg, xb, g, gamma, mean, rstd, ds)), ("dx", act)
        worst = GR.check_sums(pkg, xb, g, gamma, mean, rstd, G, dg, db, ds, info) if stats else None
        return (y, mean, rstd, dx, dr, dg, db, ds), worst
    finally:
        run.free()


# (N, HW, C, G): every Cg, C, HW and N of the module docstring
COVER = [(1, 1, 1, 1), (2, 7, 3, 3), (3, 49, 6, 3), (2, 49, 8, 2), (1, 784, 8, 1), (3, 784, 16, 1), (2, 3136, 64, 2), (128, 49, 64, 32),
         (2, 784, 256, 16), (2, 49, 320, 10), (2, 49, 320, 4), (1, 7, 2048, 1), (2, 7, 2048, 64), (3, 1, 64, 64), (1, 3136, 32, 8),
         (128, 7, 6, 6), (3, 784, 2048, 2048)]
MULTI_RANGE = [(2, 3136, 64, 2), (2, 784, 256, 16), (1, 3136, 32, 8), (3, 784, 2048, 2048)]   # several ranges per image, by design
BENCH = [(128, 3136, 64, 32), (8, 16384, 64, 32), (2, 65536, 32, 8), (16, 784, 256, 256)]


@pytest.mark.parametrize("N,HW,C,G", COVER, ids=[f"N{n}-HW{h}-C{c}-G{g}" for n, h, c, g in COVER])
def test_cover(eng, pkg, N, HW, C, G):
    """every code, with r and dy2: bit-exact y, dr and dx, statistics and sums within bounds, reruns bit-identical"""
    info = pkg.groupnorm_nhwc_info(N, HW, C, G)
    if HW > info["pixels_per_range"]:
        assert info["ranges"] >= 2, info                       # an image's pixels are split across CTAs
    if (N, HW, C, G) in MULTI_RANGE:
        assert info["ranges"] >= 4, info
    worst = {}
    for act in ACTS:
        rng = np.random.default_rng(N * 7919 + HW * 31 + C * 7 + G + act)
        xb, rb, gamma, beta, dyb, dy2b = operands(pkg, rng, N, HW, C)
        first, w = check_all(eng, pkg, xb, rb, gamma, beta, dyb, dy2b, G, act)
        for k, v in w.items():
            worst[k] = max(worst.get(k, 0.0), v)
        if act in (0, 4):
            again, _ = check_all(eng, pkg, xb, rb, gamma, beta, dyb, dy2b, G, act)
            for a, b in zip(first, again):
                assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    print(f"N{N} HW{HW} C{C} G{G}: worst ratio to bound {worst}")


@pytest.mark.parametrize("N,HW,C,G", BENCH, ids=[f"N{n}-HW{h}-C{c}-G{g}" for n, h, c, g in BENCH])
def test_benchmark_shapes(eng, pkg, N, HW, C, G):
    """the conv_bench gn shapes at their sizes: several ranges per image, more CTAs than SMs, ReLU with r and SiLU with r and dy2
    bit-exact, statistics and sums within bounds"""
    info = pkg.groupnorm_nhwc_info(N, HW, C, G)
    assert info["ranges"] >= 8 and info["ctas"] > SMS, info
    rng = np.random.default_rng(N + HW + C + G)
    xb, rb, gamma, beta, dyb, dy2b = operands(pkg, rng, N, HW, C)
    _, w3 = check_all(eng, pkg, xb, rb, gamma, beta, dyb, None, G, 3)
    _, w4 = check_all(eng, pkg, xb, rb, gamma, beta, dyb, dy2b, G, 4)
    print(f"N{N} HW{HW} C{C} G{G}: worst ratio to bound ReLU {w3} SiLU {w4}")


SPECIAL = [np.nan, np.inf, -np.inf, 0.0, -0.0]


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("C,G", [(16, 4), (6, 3)])
def test_special_values(eng, pkg, act, C, G):
    """+-0, +-Inf and NaN in x (groups 0 and, when C > 8, the group after) and in r (everywhere sparse): y, dr and dx follow the
    replays; the groups x leaves finite keep finite statistics"""
    N, HW = 2, 49
    rng = np.random.default_rng(act * 3 + C)
    xb, rb, gamma, beta, dyb, dy2b = operands(pkg, rng, N, HW, C)
    x = pkg.bf16_bits_to_f32(xb)
    x[0, :len(SPECIAL), 0] = SPECIAL                           # group 0 of image 0: NaN statistics
    x[1, 3, 0], x[1, 5, 0] = 0.0, -0.0                         # zeros only: finite statistics
    r = pkg.bf16_bits_to_f32(rb)
    r.reshape(-1)[::37] = np.resize(SPECIAL, r.reshape(-1)[::37].size)
    xb, rb = bits(pkg, x), bits(pkg, r)
    (y, mean, rstd, *_), _ = check_all(eng, pkg, xb, rb, gamma, beta, dyb, dy2b, G, act, stats=False)
    assert np.isnan(mean[0, 0]) and np.all(np.isfinite(mean[1])) and np.all(np.isfinite(mean[0, 1:]))
    fin = np.isfinite(pkg.bf16_bits_to_f32(xb)).reshape(N, HW, G, -1).all(axis=(1, 3))
    assert np.array_equal(np.isfinite(mean), fin)


def test_integer_sums_are_exact(eng, pkg):
    """small integer g (act 0, no dy2) and integer gamma: dbeta = sum g and A = sum gamma g are exact in float64"""
    N, HW, C, G = 3, 784, 16, 4
    rng = np.random.default_rng(3)
    xb, _, _, beta, _, _ = operands(pkg, rng, N, HW, C)
    gamma = rng.integers(-4, 5, C).astype(np.float32)
    dyb = bits(pkg, rng.integers(-8, 9, (N, HW, C)))
    run = Run(eng, pkg, xb, gamma, beta, G, 0)
    try:
        run.fwd()
        dx, dr, dg, db, ds = run.bwd(dyb)
    finally:
        run.free()
    g = pkg.bf16_bits_to_f32(dyb).astype(np.float64)
    assert np.array_equal(db, g.sum(axis=(0, 1)))
    assert np.array_equal(ds[0], GR.group_view(gamma * g, G).sum(axis=2))


@pytest.mark.parametrize("N,HW,C,G,act", [(128, 784, 64, 8, 3), (128, 49, 6, 3, 4), (128, 7, 320, 4, 6)])
def test_image_alone_equals_image_in_batch(eng, pkg, N, HW, C, G, act):
    """images 0, 1 and N - 1 run alone (N = 1) give the bits they get in the batch of N: y, the statistics, dstat, dx and dr"""
    rng = np.random.default_rng(N + HW + C)
    xb, rb, gamma, beta, dyb, dy2b = operands(pkg, rng, N, HW, C)
    batch, _ = check_all(eng, pkg, xb, rb, gamma, beta, dyb, dy2b, G, act, stats=False)
    y, mean, rstd, dx, dr, _, _, ds = batch
    for n in (0, 1, N - 1):
        one, _ = check_all(eng, pkg, xb[n:n + 1], rb[n:n + 1], gamma, beta, dyb[n:n + 1], dy2b[n:n + 1], G, act, stats=False)
        y1, m1, s1, dx1, dr1, _, _, ds1 = one
        assert np.array_equal(y1[0], y[n]) and np.array_equal(dx1[0], dx[n]) and np.array_equal(dr1[0], dr[n])
        assert np.array_equal(m1[0].view(np.uint32), mean[n].view(np.uint32))
        assert np.array_equal(s1[0].view(np.uint32), rstd[n].view(np.uint32))
        assert np.array_equal(ds1[:, 0].view(np.uint32), ds[:, n].view(np.uint32))


@pytest.mark.parametrize("act", [0, 3, 5])
def test_in_place_and_without_dr(eng, pkg, act):
    """dx == dy gives the out-of-place bits; dr = None and dy2 = None leave dx to the same rules"""
    N, HW, C, G = 2, 784, 24, 6
    rng = np.random.default_rng(70 + act)
    xb, rb, gamma, beta, dyb, _ = operands(pkg, rng, N, HW, C)
    run = Run(eng, pkg, xb, gamma, beta, G, act, rb)
    try:
        run.fwd()
        out = run.bwd(dyb, None, with_dr=True)
        inp = run.bwd(dyb, None, with_dr=False, in_place=True)
    finally:
        run.free()
    assert np.array_equal(out[0], inp[0]) and inp[1] is None
    for a, b in zip(out[2:], inp[2:]):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(eng, pkg):
    """every domain, act, NULL, alignment and overlap rule of the three entries is refused with PCNN_ERR_ARG and its rule"""
    N, HW, C, G = 2, 16, 16, 4
    n = N * HW * C
    x, r, y, dy, dy2, dx, dr = (eng.array(n + 64, np.uint16) for _ in range(7))
    gamma, beta, dg, db = (eng.to_device(np.ones(C + 16, np.float32)) for _ in range(4))
    sm, sr, ds = eng.array(N * G + 16), eng.array(N * G + 16), eng.array(2 * N * G + 16)
    F_, B_, P_ = "pcnn_groupnorm_nhwc_bf16_fwd", "pcnn_groupnorm_nhwc_bf16_bwd", "pcnn_groupnorm_nhwc_bf16_bwd_preact"

    def fwd(**k):
        a = dict(x=x, y=y, N=N, HW=HW, C=C, G=G, gamma=gamma, beta=beta, save_mean=sm, save_rstd=sr, r=r, act=0, eps=1e-5)
        a.update(k)
        eng.groupnorm_fwd(**a)

    def bwd(**k):
        a = dict(x=x, y=y, dy=dy, gamma=gamma, save_mean=sm, save_rstd=sr, dx=dx, dgamma=dg, dbeta=db, dstat=ds, N=N, HW=HW, C=C, G=G,
                 act=0, dy2=dy2, dr=dr)
        a.update(k)
        eng.groupnorm_bwd(**a)

    def pre(**k):
        a = dict(x=x, dy=dy, gamma=gamma, beta=beta, save_mean=sm, save_rstd=sr, dx=dx, dgamma=dg, dbeta=db, dstat=ds, N=N, HW=HW, C=C,
                 G=G, act=4, r=r, dy2=dy2, dr=dr)
        a.update(k)
        eng.groupnorm_bwd_preact(**a)

    cases = [
        (lambda: fwd(N=0), F_ + ": N = 0 images: N >= 1 is required"),
        (lambda: fwd(HW=0), "H * W >= 1 is required"),
        (lambda: fwd(C=2056, G=1), "1 <= C <= 2048 is required"),
        (lambda: fwd(C=0), "1 <= C <= 2048 is required"),
        (lambda: fwd(G=3), "1 <= G <= C with C % G == 0 is required"),
        (lambda: fwd(G=32), "1 <= G <= C with C % G == 0 is required"),
        (lambda: fwd(G=0), "1 <= G <= C with C % G == 0 is required"),
        (lambda: fwd(eps=float("nan")), "a finite eps >= 0 is required"),
        (lambda: fwd(eps=-1.0), "a finite eps >= 0 is required"),
        (lambda: fwd(eps=float("inf")), "a finite eps >= 0 is required"),
        (lambda: fwd(act=1), F_ + ": act 1 (sigmoid) is not available after group normalization"),
        (lambda: fwd(act=2), "is not 0 (none) or 3 (ReLU), nor 4 (SiLU), 5 (hard-swish) or 6 (ReLU6)"),
        (lambda: fwd(act=7), "is not 0 (none) or 3 (ReLU), nor 4 (SiLU), 5 (hard-swish) or 6 (ReLU6)"),
        (lambda: bwd(act=4), B_ + ": act 4 takes its gradient from the recomputed pre-activation"),
        (lambda: bwd(act=1), B_ + ": act 1 (sigmoid) is not available"),
        (lambda: bwd(act=2), B_ + ": act 2 is not 0 (none) or 3 (ReLU)"),
        (lambda: pre(act=0), P_ + ": act 0 takes its gradient from y"),
        (lambda: pre(act=3), P_ + ": act 3 takes its gradient from y"),
        (lambda: pre(act=7), P_ + ": act 7 is not 4 (SiLU), 5 (hard-swish) or 6 (ReLU6)"),
        (lambda: bwd(G=5), B_ + ": G = 5 groups"),
        (lambda: pre(N=0), P_ + ": N = 0 images"),
        (lambda: fwd(x=None), F_ + ": NULL context, x, y, gamma, beta, save_mean or save_rstd (only r may be NULL)"),
        (lambda: fwd(y=None), "(only r may be NULL)"),
        (lambda: fwd(beta=None), "(only r may be NULL)"),
        (lambda: fwd(save_mean=None), "(only r may be NULL)"),
        (lambda: fwd(save_rstd=None), "(only r may be NULL)"),
        (lambda: bwd(dstat=None), B_ + ": NULL context, x, y, dy, gamma, save_mean, save_rstd, dx, dgamma, dbeta or dstat"),
        (lambda: bwd(y=None), "(only dy2 and dr may be NULL)"),
        (lambda: bwd(dgamma=None), "(only dy2 and dr may be NULL)"),
        (lambda: pre(beta=None), P_ + ": NULL context, x, dy, gamma, beta, save_mean, save_rstd, dx, dgamma, dbeta or dstat"),
        (lambda: pre(dstat=None), "(only r, dy2 and dr may be NULL)"),
        (lambda: fwd(x=x.ptr + 2), F_ + ": x, r, y, gamma, beta, save_mean and save_rstd must be 16-byte aligned"),
        (lambda: fwd(r=r.ptr + 8), "must be 16-byte aligned"),
        (lambda: fwd(save_rstd=sr.ptr + 4), "must be 16-byte aligned"),
        (lambda: bwd(dstat=ds.ptr + 4), B_ + ": x, y, dy, dy2, dx, dr, gamma, dgamma, dbeta, dstat and the statistics must be 16-byte aligned"),
        (lambda: bwd(dy2=dy2.ptr + 2), "must be 16-byte aligned"),
        (lambda: pre(beta=beta.ptr + 4), P_ + ": x, r, dy, dy2, dx, dr, gamma, beta, dgamma, dbeta, dstat and the statistics must be 16-byte aligned"),
        (lambda: fwd(y=x), F_ + ": overlapping buffers: x, r, y, gamma, beta and the statistics must not share memory"),
        (lambda: fwd(save_rstd=sm.ptr + 16), "overlapping buffers"),
        (lambda: bwd(dx=dy.ptr + 16), B_ + ": overlapping buffers: only dx == dy (in place) may share memory"),
        (lambda: bwd(dr=dx), "only dx == dy (in place) may share memory"),
        (lambda: bwd(dstat=sm), "only dx == dy (in place) may share memory"),
        (lambda: pre(dx=x), P_ + ": overlapping buffers: only dx == dy (in place) may share memory"),
        (lambda: pre(dstat=dg.ptr + 16), "only dx == dy (in place) may share memory"),
    ]
    try:
        for call, msg in cases:
            with pytest.raises(pkg.PcnnError) as e:
                call()
            assert e.value.code != 0 and msg in e.value.msg, (msg, e.value.msg)
    finally:
        for a in (x, r, y, dy, dy2, dx, dr, gamma, beta, dg, db, sm, sr, ds):
            a.free()


# ------------------------------------------------------------------------------------------------ the layer
@pytest.mark.parametrize("act", ACTS)
def test_layer_step(eng, pkg, act):
    """GroupNormLayer forward with r and backward with dy2 and dr: y, dr and dx bit-exact against the replays on the layer's
    saved statistics and dstat; at codes 4-6 the layer keeps r for its backward"""
    N, H, W, C, G = 2, 6, 6, 24, 8
    rng = np.random.default_rng(80 + act)
    xb, rb, gamma, beta, dyb, dy2b = operands(pkg, rng, N, H * W, C)
    L = pkg.GroupNormLayer(eng, N, H, W, C, G, act=act, gamma=gamma, beta=beta)
    xd, rd, dyd, dy2d = (eng.to_device(a) for a in (xb, rb, dyb, dy2b))
    yd, dxd, drd = (eng.array(xb.size, np.uint16) for _ in range(3))
    try:
        L.forward(xd, yd, r=rd)
        L.backward(yd, dyd, dxd, dr=drd, dy2=dy2d)
        eng.sync()
        mean, rstd = L.save_mean.to_host().reshape(N, G), L.save_rstd.to_host().reshape(N, G)
        y = yd.to_host().reshape(xb.shape)
        assert same_or_nan(y, GR.fwd_bits(pkg, xb, gamma, beta, mean, rstd, rb, act))
        g = GR.grad_bits(pkg, xb, gamma, beta, mean, rstd, dyb, dy2b, rb if act in BA.CODES else None, act, y)
        assert same_or_nan(drd.to_host().reshape(xb.shape), g)
        ds = L.dstat.to_host()
        assert same_or_nan(dxd.to_host().reshape(xb.shape), GR.dx_bits(pkg, xb, g, gamma, mean, rstd, ds))
        GR.check_sums(pkg, xb, g, gamma, mean, rstd, G, L.dgamma.to_host(), L.dbeta.to_host(), ds, L.info)
        assert (L._r is rd) == (act in BA.CODES)
        assert L.optim_tensors()[0][4] and len(L.params()) == 2
    finally:
        for a in (xd, rd, dyd, dy2d, yd, dxd, drd):
            a.free()
        L.close()


@pytest.mark.parametrize("kind", ["sgd", "adamw"])
def test_optimizers(eng, pkg, kind):
    """pkg.SGD (momentum, decay) and pkg.AdamW over a SiLU GroupNormLayer, bit-identical to the float32 replays over 3 steps"""
    N, H, W, C, G = 2, 5, 5, 16, 4
    rng = np.random.default_rng(9)
    xb, rb, gamma, beta, dyb, _ = operands(pkg, rng, N, H * W, C)
    L = pkg.GroupNormLayer(eng, N, H, W, C, G, act=pkg.ACT_SILU, gamma=gamma, beta=beta)
    xd, rd, dyd = eng.to_device(xb), eng.to_device(rb), eng.to_device(dyb)
    yd, dxd = eng.array(xb.size, np.uint16), eng.array(xb.size, np.uint16)
    opt = pkg.SGD(eng, [L], momentum=0.9, weight_decay=1e-2) if kind == "sgd" else pkg.AdamW(eng, [L], weight_decay=1e-2)
    tensors = L.optim_tensors()
    state = [[None, np.zeros(C, np.float32), np.zeros(C, np.float32)] for _ in tensors]
    try:
        for t in range(1, 4):
            lr = 0.05 * t
            L.forward(xd, yd, r=rd)
            L.backward(yd, dyd, dxd)
            eng.sync()
            ps, gs = [p.to_host().reshape(-1) for p, *_ in tensors], [g.to_host().reshape(-1) for _, g, *_ in tensors]
            assert all(np.isfinite(g).all() for g in gs)
            opt.step(lr)
            eng.sync()
            for i, (p, g) in enumerate(zip(ps, gs)):
                if kind == "sgd":
                    want, state[i][0] = OR.sgd32(p, g, state[i][0], lr, t, momentum=0.9, wd=1e-2)
                else:
                    want, state[i][1], state[i][2] = OR.adamw32(p, g, state[i][1], state[i][2], lr, t, wd=1e-2)
                assert np.array_equal(tensors[i][0].to_host().reshape(-1).view(np.uint32), want.view(np.uint32)), (kind, t, i)
    finally:
        opt.close()
        for a in (xd, rd, dyd, yd, dxd):
            a.free()
        L.close()
