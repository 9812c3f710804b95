"""SiLU, hard-swish and ReLU6 after batch normalization (pcnn_batchnorm_nhwc_bf16_fwd at codes 4-6, and
pcnn_batchnorm_nhwc_bf16_bwd_preact): y, g (= dr) and dx bit for bit against the float32 replays of bnact_ref.py and
batchnorm_ref.py on the device's own statistics and gradient sums, with operands built so that the pre-activation hits every
branch, knee and special value; dgamma and dbeta within batchnorm_ref.n_acc's bound; buffers, in-place calls, reruns and
refusals; a BatchNormLayer step at each code with SGD and AdamW over it; and an EfficientNet-style network trained on MNIST
digits, checked bit for bit at every new-code BN in its first steps."""
import numpy as np
import pytest

import batchnorm_ref as BR
import bnact_ref as AR
import optim_ref as OR
from batchnorm_ref import U, n_acc
from example_nets import NAN_BF16, EfficientNetLite, host, train

pytestmark = pytest.mark.gpu

TAIL = 64
IDS = {c: AR.NAMES[c] for c in AR.CODES}

CS_ = [1, 3, 6, 8, 16, 64, 120, 256]
PIXELS = [2, 7, 1001]
GRID = [(C, p) for C in CS_ for p in PIXELS] + [(64, 128 * 56 * 56)]
GIDS = [f"C{C}-px{p}" for C, p in GRID]
# r values of the special channel (gamma = +0 and beta = -0 there, so v = r exactly): every knee, both zeros, the E thresholds and
# overflow, the bf16 band below 6, infinities and NaN
SPECIAL_R = [np.nan, np.inf, -np.inf, 0.0, -0.0, -3.0, 3.0, 6.0, -6.0, 5.96875, 2.984375, -2.984375, -1.5, -1.28125, 1.0, -1.0,
             -88.5, -89.0, -100.0, -104.0, -110.0, 88.5, 89.0, 100.0, 1e30, -1e30, 3.0e38, -3.0e38]


def bits(pkg, a):
    return pkg.f32_to_bf16_bits(np.asarray(a, np.float32))


def same_or_nan(got, want):
    """bf16 bits: identical where want is a number; NaN (any payload) where want is NaN"""
    got, want = np.asarray(got, np.uint16), np.asarray(want, np.uint16)
    nan, gnan = (want & 0x7FFF) > 0x7F80, (got & 0x7FFF) > 0x7F80
    return np.array_equal(gnan, nan) and np.array_equal(got[~nan], want[~nan])


class Stats:
    def __init__(self, eng, gamma, beta, rm, rv):
        C = gamma.size
        self.gamma, self.beta = eng.to_device(np.asarray(gamma, np.float32)), eng.to_device(np.asarray(beta, np.float32))
        self.rm, self.rv = eng.to_device(np.asarray(rm, np.float32)), eng.to_device(np.asarray(rv, np.float32))
        self.sm, self.sr = eng.to_device(np.full(C, np.nan, np.float32)), eng.to_device(np.full(C, np.nan, np.float32))

    def free(self):
        for a in (self.gamma, self.beta, self.rm, self.rv, self.sm, self.sr):
            a.free()


def operands(pkg, rng, pixels, C, special=True):
    """x with a spread per channel, gamma up to 4 and beta in (-4, 7) so that v crosses every knee; r wide; with C > 1 and
    `special`, channel 0 has gamma = +0, beta = -0 and r cycling through SPECIAL_R, so that its v is exactly those values (-0
    included, at the pixels where xhat < 0)"""
    x = rng.standard_normal((pixels, C)) * rng.uniform(0.5, 2, C) + rng.uniform(-4, 4, C)
    gamma, beta = rng.uniform(0.5, 4, C), rng.uniform(-4, 7, C)
    r = rng.standard_normal((pixels, C)) * 4
    r[rng.random((pixels, C)) < 0.02] = -95.0                     # SiLU's E overflow in every channel
    if special and C > 1:
        gamma[0], beta[0] = 0.0, -0.0                             # RN(xhat * 0) + (-0) is -0 where xhat < 0, so r = -0 gives v = -0
        r[:, 0] = np.resize(SPECIAL_R, pixels)
    rm, rv = rng.uniform(-1, 1, C), rng.uniform(0.5, 2, C)
    return bits(pkg, x), bits(pkg, r), gamma.astype(np.float32), beta.astype(np.float32), rm.astype(np.float32), rv.astype(np.float32)


def run_fwd(eng, xb, rb, st, act, training):
    pixels, C = xb.shape
    xd = eng.to_device(xb)
    rd = None if rb is None else eng.to_device(rb)
    y = eng.to_device(np.full(pixels * C + TAIL, NAN_BF16, np.uint16))
    eng.batchnorm_fwd(xd, y, pixels, C, st.gamma, st.beta, st.rm, st.rv, st.sm, st.sr, r=rd, act=act, training=training)
    eng.sync()
    out = y.to_host()
    for a in (xd, rd, y):
        if a is not None:
            a.free()
    return out


def run_bwd(eng, xb, rb, dyb, st, act, dy2b=None, with_dr=True, in_place=False):
    pixels, C = xb.shape
    n = pixels * C
    xd = eng.to_device(xb)
    rd = None if rb is None else eng.to_device(rb)
    dyd = eng.to_device(np.concatenate([dyb.reshape(-1), np.full(TAIL, NAN_BF16, np.uint16)]))
    dy2d = None if dy2b is None else eng.to_device(dy2b)
    dx = dyd if in_place else eng.to_device(np.full(n + TAIL, NAN_BF16, np.uint16))
    dr = eng.to_device(np.full(n + TAIL, NAN_BF16, np.uint16)) if with_dr else None
    dg, db = eng.to_device(np.full(C, np.nan, np.float32)), eng.to_device(np.full(C, np.nan, np.float32))
    eng.batchnorm_bwd_preact(xd, dyd, st.gamma, st.beta, st.sm, st.sr, dx, dg, db, pixels, C, act, r=rd, dy2=dy2d, dr=dr)
    eng.sync()
    out = dx.to_host(), (dr.to_host() if with_dr else None), dg.to_host(), db.to_host()
    for a in {id(v): v for v in (xd, rd, dyd, dy2d, dx, dr, dg, db) if v is not None}.values():
        a.free()
    return out


def check_sums(pkg, g, xb, mean, rstd, dg, db):
    """dbeta and dgamma within 2 (n_acc + 1) u sum |term| of float64 over the replayed g; NaN exactly where float64 is NaN"""
    pixels, C = xb.shape
    gf = pkg.bf16_bits_to_f32(g).astype(np.float64)
    xh = BR.xhat32(pkg, xb, mean, rstd).astype(np.float64)
    na = n_acc(pkg, pixels, C)
    with np.errstate(invalid="ignore"):
        for got, terms in ((db, gf), (dg, gf * xh)):
            want = terms.sum(0)
            nan = np.isnan(want)
            assert np.array_equal(np.isnan(got), nan)
            assert np.all(np.abs(got[~nan] - want[~nan]) <= 2 * (na + 1) * U * np.abs(terms).sum(0)[~nan])


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("C,pixels", GRID, ids=GIDS)
def test_forward(eng, pkg, C, pixels):
    """codes 4-6, training and eval, with and without r: y bit-identical to the replay (NaN where it is NaN), NaN-prefilled y
    fully written with its tail untouched, saved statistics as at act 0, reruns bit-identical"""
    rng = np.random.default_rng(C * 1013 + pixels)
    xb, rb, gamma, beta, rm0, rv0 = operands(pkg, rng, pixels, C)
    n = pixels * C
    for act in AR.CODES:
        for with_r in (True, False):
            r = rb if with_r else None
            for training in (True, False):
                st = Stats(eng, gamma, beta, rm0, rv0)
                y = run_fwd(eng, xb, r, st, act, training)
                assert np.all(y[n:] == NAN_BF16)
                if training:
                    mean, rstd = st.sm.to_host(), st.sr.to_host()
                    ref = Stats(eng, gamma, beta, rm0, rv0)
                    run_fwd(eng, xb, r, ref, 0, True)
                    assert np.array_equal(mean.view(np.uint32), ref.sm.to_host().view(np.uint32))
                    assert np.array_equal(rstd.view(np.uint32), ref.sr.to_host().view(np.uint32))
                    ref.free()
                else:
                    mean, rstd = rm0, BR.eval_rstd(rv0, 1e-5)
                v = AR.pre32(pkg, xb, gamma, beta, mean, rstd, r)
                assert same_or_nan(y[:n].reshape(pixels, C), AR.act_bits(pkg, v, act)), (IDS[act], with_r, training)
                if with_r and C > 1 and pixels >= len(SPECIAL_R):      # the special channel took every listed v
                    want_v = pkg.bf16_bits_to_f32(bits(pkg, SPECIAL_R[1:]))
                    assert np.isin(want_v, v[:, 0]).all() and np.isnan(v[:, 0]).any()
                    v0 = v[:, 0]
                    assert np.any((v0 == 0) & ~np.signbit(v0))
                    if training:                                        # xhat < 0 at about half the pixels: v = -0 reaches the device
                        assert np.any((v0 == 0) & np.signbit(v0))
                if training and with_r:
                    again = run_fwd(eng, xb, r, st, act, training)
                    assert np.array_equal(again, y)
                st.free()


# ------------------------------------------------------------------------------------------------ backward
@pytest.mark.parametrize("C,pixels", GRID, ids=GIDS)
def test_backward(eng, pkg, C, pixels):
    """codes 4-6, with and without r and dy2: dr bit-identical to the replayed g at the recomputed v, dx bit-identical to the
    replay from the device's dgamma, dbeta and statistics, the sums within bound, NaN-prefilled outputs fully written with tails
    untouched; in place equals out of place; reruns bit-identical"""
    rng = np.random.default_rng(C * 37 + pixels)
    xb, rb, gamma, beta, rm0, rv0 = operands(pkg, rng, pixels, C)
    n = pixels * C
    dyb = bits(pkg, rng.standard_normal((pixels, C)))
    dy2b = bits(pkg, rng.standard_normal((pixels, C)))
    for act in AR.CODES:
        combos = [(wr, d2) for wr in (True, False) for d2 in (None, dy2b)]
        for with_r, d2 in combos:
            r = rb if with_r else None
            st = Stats(eng, gamma, beta, rm0, rv0)
            run_fwd(eng, xb, r, st, act, True)
            mean, rstd = st.sm.to_host(), st.sr.to_host()
            dx, dr, dg, db = run_bwd(eng, xb, r, dyb, st, act, d2)
            assert np.all(dx[n:] == NAN_BF16) and np.all(dr[n:] == NAN_BF16)
            v = AR.pre32(pkg, xb, gamma, beta, mean, rstd, r)
            g = AR.grad_bits(pkg, v, dyb, d2, act)
            assert same_or_nan(dr[:n].reshape(pixels, C), g), (IDS[act], with_r, d2 is None)
            check_sums(pkg, g, xb, mean, rstd, dg, db)
            with np.errstate(all="ignore"):
                want = BR.dx_bits(pkg, xb, g, gamma, mean, rstd, dg, db)
            assert same_or_nan(dx[:n].reshape(pixels, C), want), (IDS[act], with_r, d2 is None)
            if d2 is None and with_r:                                # in place and a rerun, once per code
                ip = run_bwd(eng, xb, r, dyb, st, act, None, with_dr=False, in_place=True)
                assert np.array_equal(ip[0], dx) and np.array_equal(ip[2].view(np.uint32), dg.view(np.uint32))
                again = run_bwd(eng, xb, r, dyb, st, act, None)
                assert all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(again, (dx, dr, dg, db)))
            st.free()


def test_relu6_band_and_r_matter(eng, pkg):
    """v in (5.984, 6), which bf16 rounds to y = 6: the device passes the gradient there (a mask from y would cut it), and a
    backward handed no r where the forward had one gives a different dx"""
    pixels, C = 4096, 8
    rng = np.random.default_rng(3)
    xb, rb, gamma, beta, rm0, rv0 = operands(pkg, rng, pixels, C, special=False)
    gamma[:] = 0.0
    beta[:] = 5.99                                                  # v = 5.99 + r, r small: many v in the band
    rb = bits(pkg, rng.uniform(-0.02, 0.02, (pixels, C)))
    st = Stats(eng, gamma, beta, rm0, rv0)
    y = run_fwd(eng, xb, rb, st, AR.RELU6, True)[:pixels * C].reshape(pixels, C)
    v = AR.pre32(pkg, xb, gamma, beta, st.sm.to_host(), st.sr.to_host(), rb)
    band = (v > 5.984375) & (v < 6)
    assert band.sum() > 100 and np.all(pkg.bf16_bits_to_f32(y[band]) == 6)
    dyb = bits(pkg, rng.standard_normal((pixels, C)))
    dx, dr, dg, db = run_bwd(eng, xb, rb, dyb, st, AR.RELU6)
    assert np.array_equal(dr[:pixels * C].reshape(pixels, C)[band], dyb[band])
    dx0 = run_bwd(eng, xb, None, dyb, st, AR.RELU6)[0]
    assert not np.array_equal(dx0, dx)
    st.free()


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(eng, pkg):
    pixels, C = 64, 16
    n = pixels * C
    t = [eng.array(n + 64, np.uint16) for _ in range(7)]
    x, r, y, dy, dy2, dx, dr = t
    v = [eng.array(C + 8) for _ in range(8)]
    gamma, beta, rm, rv, sm, sr, dg, db = v
    fwd = lambda **kw: eng.batchnorm_fwd(**{**dict(x=x, y=y, pixels=pixels, C=C, gamma=gamma, beta=beta, running_mean=rm, running_var=rv,
                                                   save_mean=sm, save_rstd=sr, r=r, act=4, training=True), **kw})
    old = lambda **kw: eng.batchnorm_bwd(**{**dict(x=x, y=y, dy=dy, gamma=gamma, save_mean=sm, save_rstd=sr, dx=dx, dgamma=dg, dbeta=db,
                                                   pixels=pixels, C=C, act=3, dy2=None, dr=dr), **kw})
    pre = lambda **kw: eng.batchnorm_bwd_preact(**{**dict(x=x, dy=dy, gamma=gamma, beta=beta, save_mean=sm, save_rstd=sr, dx=dx, dgamma=dg,
                                                          dbeta=db, pixels=pixels, C=C, act=4, r=r, dy2=dy2, dr=dr), **kw})
    F, B, P = "pcnn_batchnorm_nhwc_bf16_fwd", "pcnn_batchnorm_nhwc_bf16_bwd", "pcnn_batchnorm_nhwc_bf16_bwd_preact"
    esc = lambda s: s.replace("(", r"\(").replace(")", r"\)").replace("*", r"\*").replace("+", r"\+")
    cases = [
        (lambda: fwd(act=2), F + ": act 2 is not 0 (none) or 3 (ReLU), nor 4 (SiLU), 5 (hard-swish) or 6 (ReLU6)"),
        (lambda: fwd(act=7), F + ": act 7 is not 0 (none) or 3 (ReLU)"),
        (lambda: fwd(act=1), F + ": act 1 (sigmoid) is not available after batch normalization: sigmoid_bf16 uses tanh.approx, which no "
                                 "reference can replay bit for bit; act 0 (none) or 3 (ReLU) is required"),
        (lambda: old(act=4), B + ": act 4 takes its gradient from the recomputed pre-activation, not from y: " + P),
        (lambda: old(act=5), B + ": act 5 takes its gradient"),
        (lambda: old(act=6), B + ": act 6 takes its gradient"),
        (lambda: old(act=7), B + ": act 7 is not 0 (none) or 3 (ReLU)"),
        (lambda: pre(act=0), P + ": act 0 takes its gradient from y: " + B + " is its backward"),
        (lambda: pre(act=3), P + ": act 3 takes its gradient from y"),
        (lambda: pre(act=1), P + ": act 1 (sigmoid) is not available after batch normalization: sigmoid_bf16 uses tanh.approx, which no "
                                 "reference can replay bit for bit; act 4 (SiLU), 5 (hard-swish) or 6 (ReLU6) is required"),
        (lambda: old(act=1), B + ": act 1 (sigmoid) is not available after batch normalization: sigmoid_bf16 uses tanh.approx, which no "
                                 "reference can replay bit for bit; act 0 (none) or 3 (ReLU) is required"),
        (lambda: pre(act=2), P + ": act 2 is not 4 (SiLU), 5 (hard-swish) or 6 (ReLU6)"),
        (lambda: pre(act=7), P + ": act 7 is not 4 (SiLU)"),
        (lambda: pre(C=0), P + ": C = 0 channels: 1 <= C <= 256 is required"),
        (lambda: pre(C=257), P + ": C = 257 channels"),
        (lambda: pre(pixels=1), P + ": pixels = 1: training needs more than 1 value per channel"),
        (lambda: fwd(C=300), F + ": C = 300 channels"),
        (lambda: pre(x=None), P + ": NULL context, x, dy, gamma, beta, save_mean, save_rstd, dx, dgamma or dbeta"),
        (lambda: pre(dy=None), "NULL context, x, dy, gamma, beta"),
        (lambda: pre(beta=None), "NULL context, x, dy, gamma, beta"),
        (lambda: pre(gamma=None), "NULL context, x, dy, gamma, beta"),
        (lambda: pre(dx=None), "NULL context, x, dy, gamma, beta"),
        (lambda: pre(dbeta=None), "NULL context, x, dy, gamma, beta"),
        (lambda: pre(save_rstd=None), "NULL context, x, dy, gamma, beta"),
        (lambda: pre(x=x.ptr + 2), P + ": x, r, dy, dy2, dx, dr, gamma, beta, dgamma, dbeta and the statistics must be 16-byte aligned"),
        (lambda: pre(r=r.ptr + 8), "must be 16-byte aligned"),
        (lambda: pre(beta=beta.ptr + 4), "must be 16-byte aligned"),
        (lambda: pre(dx=dy.ptr + 16), P + ": overlapping buffers: only dx == dy (in place) may share memory"),
        (lambda: pre(dx=x), "only dx == dy (in place) may share memory"),
        (lambda: pre(dx=r), "only dx == dy (in place) may share memory"),
        (lambda: pre(dr=r), "only dx == dy (in place) may share memory"),
        (lambda: pre(dr=dy), "only dx == dy (in place) may share memory"),
        (lambda: pre(dy2=dy), "only dx == dy (in place) may share memory"),
        (lambda: pre(dbeta=beta), "only dx == dy (in place) may share memory"),
        (lambda: pre(dgamma=gamma), "only dx == dy (in place) may share memory"),
    ]
    for fn, msg in cases:
        with pytest.raises(pkg.PcnnError, match=esc(msg)):
            fn()
    for act in AR.CODES:
        fwd(act=act)
        fwd(act=act, r=None, training=False)
        pre(act=act, r=None, dy2=None, dr=None)
        pre(act=act, dx=dy, dr=None)                                     # in place
    eng.sync()
    for a in t + v:
        a.free()


# ------------------------------------------------------------------------------------------------ layer
@pytest.mark.parametrize("act", AR.CODES, ids=[IDS[c] for c in AR.CODES])
def test_layer_step(eng, pkg, act):
    """BatchNormLayer at each code, forward with r and backward with dy2 and dr: y, dr and dx bit-exact against the replays on the
    device's statistics, and the layer keeps r for its backward; at codes 0 and 3 nothing of this applies (the old entry)"""
    N, H, W, C = 4, 6, 6, 24
    M = N * H * W
    rng = np.random.default_rng(act)
    xb, rb, gamma, beta, _, _ = operands(pkg, rng, M, C, special=False)
    L = pkg.BatchNormLayer(eng, N, H, W, C, act=act, gamma=gamma, beta=beta)
    d = lambda a: eng.to_device(a)
    xd, rd = d(xb), d(rb)
    dyb, dy2b = bits(pkg, rng.standard_normal((M, C))), bits(pkg, rng.standard_normal((M, C)))
    yd, dyd, dy2d, dxd, drd = d(np.full(M * C, NAN_BF16, np.uint16)), d(dyb), d(dy2b), d(np.full(M * C, NAN_BF16, np.uint16)), \
        d(np.full(M * C, NAN_BF16, np.uint16))
    L.forward(xd, yd, r=rd)
    L.backward(yd, dyd, dxd, dr=drd, dy2=dy2d)
    eng.sync()
    mean, rstd = L.save_mean.to_host(), L.save_rstd.to_host()
    v = AR.pre32(pkg, xb, gamma, beta, mean, rstd, rb)
    assert same_or_nan(yd.to_host().reshape(M, C), AR.act_bits(pkg, v, act))
    g = AR.grad_bits(pkg, v, dyb, dy2b, act)
    assert np.array_equal(drd.to_host().reshape(M, C), g)
    assert np.array_equal(dxd.to_host().reshape(M, C), BR.dx_bits(pkg, xb, g, gamma, mean, rstd, L.dgamma.to_host(), L.dbeta.to_host()))
    for a in (xd, rd, yd, dyd, dy2d, dxd, drd):
        a.free()
    L.close()


@pytest.mark.parametrize("kind", ["sgd", "adamw"])
def test_optimizers(eng, pkg, kind):
    """pkg.SGD (momentum, decay) and pkg.AdamW over a SiLU BatchNormLayer, bit-identical to the float32 replays over 3 steps"""
    N, H, W, C = 4, 5, 5, 16
    M = N * H * W
    rng = np.random.default_rng(9)
    xb, rb, gamma, beta, _, _ = operands(pkg, rng, M, C, special=False)
    L = pkg.BatchNormLayer(eng, N, H, W, C, act=pkg.ACT_SILU, gamma=gamma, beta=beta)
    xd, rd, dyd = eng.to_device(xb), eng.to_device(rb), eng.to_device(bits(pkg, rng.standard_normal((M, C))))
    yd, dxd = eng.array(M * C, np.uint16), eng.array(M * C, np.uint16)
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
        L.close()
        for a in (xd, rd, dyd, yd, dxd):
            a.free()


# ------------------------------------------------------------------------------------------------ end to end
ACC_MIN = 0.85          # the float32 torch CPU replica (scripts/efficientnet_replica.py) of this network reaches 0.902 (DESIGN 3.20)


def test_efficientnet_mnist(eng, pkg, golden):
    """In each of the first 5 steps every new-code BN's y, g (dr) and dx are bit-exact against the replays on the device's own x,
    dy, statistics and gradient sums.  A second fresh run reproduces the parameters after 5 steps bit for bit.  After EPOCHS epochs
    over the 1024 training digits the mean loss has fallen, and test accuracy on the 256 test digits, evaluated with the running
    statistics, exceeds ACC_MIN."""

    def check_step(net, it, x, labels):
        net.forward(x, labels)
        net.backward()
        eng.sync()
        for bn, x, y, dy, dx, g in net.bn_tensors():
            C = bn.shape[3]
            ga, be = bn.gamma.to_host(), bn.beta.to_host()
            mean, rstd = bn.save_mean.to_host(), bn.save_rstd.to_host()
            xb, yb, dyb = host(x).reshape(-1, C), host(y).reshape(-1, C), host(dy).reshape(-1, C)
            v = AR.pre32(pkg, xb, ga, be, mean, rstd)
            assert np.array_equal(yb, AR.act_bits(pkg, v, bn.act)), (it, IDS[bn.act], C)
            gb = AR.grad_bits(pkg, v, dyb, None, bn.act)
            assert np.array_equal(host(g).reshape(-1, C), gb), (it, IDS[bn.act], C)
            want = BR.dx_bits(pkg, xb, gb, ga, mean, rstd, bn.dgamma.to_host(), bn.dbeta.to_host())
            assert np.array_equal(host(dx).reshape(-1, C), want), (it, IDS[bn.act], C)

    ep_loss, acc, _ = train(eng, pkg, golden, lambda: EfficientNetLite(eng, pkg, EfficientNetLite.init_params()), EfficientNetLite.EPOCHS,
                            check_step=check_step)
    print(f"EfficientNet-style network: mean loss by epoch {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}; test accuracy {acc:.4f} (threshold {ACC_MIN})")
    assert np.isfinite(ep_loss).all() and ep_loss[-1] < ep_loss[0]
    assert acc > ACC_MIN
