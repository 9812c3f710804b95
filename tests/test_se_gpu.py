"""Squeeze-and-excitation on the device (pcnn_se_scale_nhwc_bf16_fwd / _bwd_gate / _bwd_input, SqueezeExcitationLayer): y, g and dx
bit-identical to the float32 replays of tests/se_ref.py (pinned to torch's CPU float64 by test_se_cpu.py), ds exact on integer
operands and bit-identical to the replay in the reported partition order on random ones, every refusal, one layer step on its own
operands, the fused optimizers over the layer, and an SE-ResNet trained on MNIST digits."""
import numpy as np
import pytest

import optim_ref as OR
import se_ref as SR
from example_nets import NAN_BF16, SEResNet, host, train

pytestmark = pytest.mark.gpu
TAIL = 64                 # elements past every output, NaN before the call and after it


def same_or_nan(got, want):
    """bf16 bits: identical where want is a number; NaN (any payload) where want is NaN"""
    nan, gnan = (want & 0x7FFF) > 0x7F80, (got & 0x7FFF) > 0x7F80
    return np.array_equal(gnan, nan) and np.array_equal(got[~nan], want[~nan])


def special(rng, shape, lo=None):
    """normal (or uniform [lo, 1)) values with NaN, +-Inf and +-0 sprinkled in"""
    a = (rng.standard_normal(shape) if lo is None else rng.uniform(lo, 1, shape)).astype(np.float32)
    flat = a.reshape(-1)
    for v, frac in ((np.nan, 0.01), (np.inf, 0.01), (-np.inf, 0.01), (0.0, 0.03), (-0.0, 0.03)):
        flat[rng.choice(flat.size, max(1, int(frac * flat.size)), replace=False)] = v
    return a


class Bufs:
    """device buffers of bf16 bits with TAIL NaN elements past each; read() checks the tail"""

    def __init__(self, eng):
        self.eng = eng

    def put(self, bits):
        return self.eng.to_device(np.concatenate([np.ascontiguousarray(bits, np.uint16).reshape(-1), np.full(TAIL, NAN_BF16, np.uint16)]))

    def out(self, n):
        return self.eng.to_device(np.full(n + TAIL, NAN_BF16, np.uint16))

    def read(self, d, shape):
        self.eng.sync()
        h = d.to_host()
        n = int(np.prod(shape))
        assert np.all(h[n:] == NAN_BF16), "written past the tensor"
        return h[:n].reshape(shape)


SHAPES = [(3 if C <= 320 else 2, H, W, C) for C in (1, 3, 6, 8, 16, 64, 256, 320, 2048) for H, W in ((1, 1), (7, 7), (56, 56))]
SHAPES.append((128, 56, 56, 64))


@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
def test_passes(eng, pkg, shape):
    N, H, W, C = shape
    HW = H * W
    info = pkg.se_scale_nhwc_info(N, H, W, C)
    rng = np.random.default_rng(sum(shape))
    bits, val = pkg.f32_to_bf16_bits, pkg.bf16_bits_to_f32
    B = Bufs(eng)
    n = N * HW * C
    x, dy, yb = (bits(special(rng, shape)) for _ in range(3))
    r, dy2 = (bits(rng.standard_normal(shape).astype(np.float32)) for _ in range(2))
    s = bits(special(rng, (N, C), lo=0.0))
    x_, s_, r_, dy_, dy2_, y_ = (B.put(a) for a in (x, s, r, dy, dy2, yb))
    xv, sv, rv, dyv, dy2v, yv = (val(a) for a in (x, s, r, dy, dy2, yb))

    # forward, with and without r, act 0 and 3
    for act in (0, 3):
        for with_r in (False, True):
            y = B.out(n)
            eng.se_scale_fwd(x_, s_, y, N, H, W, C, r=r_ if with_r else None, act=act)
            got = B.read(y, shape)
            want = bits(SR.fwd(xv, sv, rv if with_r else None, act))
            assert same_or_nan(got, want), ("fwd", act, with_r, int(np.sum(got != want)))
            if act == 3 and with_r:
                y2 = B.out(n)
                eng.se_scale_fwd(x_, s_, y2, N, H, W, C, r=r_, act=act)
                assert np.array_equal(B.read(y2, shape), got)                                        # rerun

    # gate gradient: g bit-exact, ds bit-identical to the ordered replay
    gates = {}
    for act, with_dy2 in ((0, False), (0, True), (3, False), (3, True)):
        g, ds = B.out(n), B.out(N * C)
        eng.se_scale_bwd_gate(x_, y_ if act == 3 else None, dy_, g, ds, N, H, W, C, dy2=dy2_ if with_dy2 else None, act=act)
        gg, dd = B.read(g, shape), B.read(ds, (N, C))
        want_g = SR.gate_g(dyv, yv, dy2v if with_dy2 else None, act)
        assert same_or_nan(gg, bits(want_g)), ("g", act, with_dy2)
        if not with_dy2 and act == 0:
            assert np.array_equal(gg, dy)                                                            # dy's bits pass
        want_ds = bits(SR.gate_ds(val(gg), xv, info))
        assert same_or_nan(dd, want_ds), ("ds", act, with_dy2, int(np.sum(dd != want_ds)))
        gates[(act, with_dy2)] = (gg, dd)
    g2, ds2 = B.out(n), B.out(N * C)
    eng.se_scale_bwd_gate(x_, y_, dy_, g2, ds2, N, H, W, C, dy2=dy2_, act=3)
    assert np.array_equal(B.read(g2, shape), gates[(3, True)][0]) and np.array_equal(B.read(ds2, (N, C)), gates[(3, True)][1])
    dyc = B.put(dy)                                                                                  # in place: g == dy
    eng.se_scale_bwd_gate(x_, y_, dyc, dyc, ds2, N, H, W, C, dy2=dy2_, act=3)
    assert np.array_equal(B.read(dyc, shape), gates[(3, True)][0]) and np.array_equal(B.read(ds2, (N, C)), gates[(3, True)][1])

    # integer operands: ds exact
    xi = bits(rng.integers(-4, 5, shape).astype(np.float32))
    di = bits(rng.integers(-3, 4, shape).astype(np.float32))
    g, ds = B.out(n), B.out(N * C)
    eng.se_scale_bwd_gate(B.put(xi), None, B.put(di), g, ds, N, H, W, C)
    exact = (val(di).astype(np.float64) * val(xi)).sum(axis=(1, 2))
    dd = B.read(ds, (N, C))
    assert np.array_equal(val(dd), val(bits(exact.astype(np.float32))))               # a sum of zeros may be -0 (0 * -4 first)
    assert np.array_equal(dd, bits(SR.gate_ds(val(di), val(xi), info)))               # and the replay has its sign
    assert np.array_equal(B.read(g, shape), di)

    # input gradient, without and with a pitched dpool holding specials; NaN in dpool's pad changes no bit
    gg = gates[(3, True)][0]
    g_ = B.put(gg)
    pitch = (C + 7) // 8 * 8 + 8
    dp = bits(special(rng, (N, C)))
    dpool = np.full((N, pitch), NAN_BF16, np.uint16)
    dpool[:, :C] = dp
    for with_dp in (False, True):
        dx = B.out(n)
        eng.se_scale_bwd_input(g_, s_, dx, N, H, W, C, dpool=B.put(dpool) if with_dp else None, dpool_row_pitch=pitch)
        got = B.read(dx, shape)
        want = bits(SR.dx(val(gg), sv, val(dp) if with_dp else None, HW))
        assert same_or_nan(got, want), ("dx", with_dp, int(np.sum(got != want)))
    dpool[:, C:] = 0
    dx2 = B.out(n)
    eng.se_scale_bwd_input(g_, s_, dx2, N, H, W, C, dpool=B.put(dpool), dpool_row_pitch=pitch)
    assert np.array_equal(B.read(dx2, shape), got)
    eng.se_scale_bwd_input(g_, s_, g_, N, H, W, C, dpool=B.put(dpool), dpool_row_pitch=pitch)   # in place: dx == g
    assert np.array_equal(B.read(g_, shape), got)
    print(f"SE {shape}: vec {info['vec']}, {info['ranges']} ranges, {info['ctas']} gate CTAs, n_acc {info['n_acc']}")


def test_refusals(eng, pkg):
    N, H, W, C = 2, 8, 8, 16
    B = Bufs(eng)
    n = N * H * W * C
    x, y, dy, g, dx = (B.out(n) for _ in range(5))
    s, ds, dp = B.out(N * C), B.out(N * C), B.out(N * 24)
    fwd, gate, inp = eng.se_scale_fwd, eng.se_scale_bwd_gate, eng.se_scale_bwd_input
    sh = (N, H, W, C)
    cases = [
        (lambda: fwd(x, s, y, 0, H, W, C), "pcnn_se_scale_nhwc_bf16_fwd: N = 0, H = 8, W = 8, C = 16: each must be >= 1"),
        (lambda: fwd(x, s, y, N, H, W, 0), "each must be >= 1"),
        (lambda: fwd(x, s, y, N, 46341, 46341, 1), "pcnn_se_scale_nhwc_bf16_fwd: one 46341x46341x1 image exceeds the 32-bit index range"),
        (lambda: fwd(x, s, y, *sh, act=1), "pcnn_se_scale_nhwc_bf16_fwd: act 1 \\(sigmoid\\) is not available"),
        (lambda: fwd(x, s, y, *sh, act=2), "act 2 is not 0 \\(none\\) or 3 \\(ReLU\\)"),
        (lambda: fwd(None, s, y, *sh), "NULL context, x, s or y"),
        (lambda: fwd(x, None, y, *sh), "NULL context, x, s or y"),
        (lambda: fwd(x.ptr + 2, s, y, *sh), "x, s, r and y must be 16-byte aligned"),
        (lambda: fwd(x, s.ptr + 8, y, *sh), "16-byte aligned"),
        (lambda: fwd(x, s, y, *sh, r=dy.ptr + 4), "16-byte aligned"),
        (lambda: fwd(x, s, x, *sh), "pcnn_se_scale_nhwc_bf16_fwd: overlapping buffers"),
        (lambda: fwd(x, s, y, *sh, r=y), "overlapping buffers"),
        (lambda: fwd(x, x.ptr + 32, y, *sh), "overlapping buffers"),
        (lambda: gate(x, y, dy, g, ds, 0, H, W, C), "pcnn_se_scale_nhwc_bf16_bwd_gate: N = 0"),
        (lambda: gate(x, None, dy, g, ds, *sh, act=3), "pcnn_se_scale_nhwc_bf16_bwd_gate: act 3 \\(ReLU\\) needs y"),
        (lambda: gate(x, y, dy, g, ds, *sh, act=1), "act 1 \\(sigmoid\\) is not available"),
        (lambda: gate(x, y, dy, g, ds, *sh, act=4), "act 4 is not 0"),
        (lambda: gate(None, y, dy, g, ds, *sh), "NULL context, x, dy, g or ds"),
        (lambda: gate(x, y, dy, g, None, *sh), "NULL context, x, dy, g or ds"),
        (lambda: gate(x, y, dy, g.ptr + 2, ds, *sh), "x, y, dy, dy2, g and ds must be 16-byte aligned"),
        (lambda: gate(x, y, dy, g, ds, *sh, dy2=dx.ptr + 8), "16-byte aligned"),
        (lambda: gate(x, y, dy, x, ds, *sh), "only g == dy \\(in place\\) may share memory"),
        (lambda: gate(x, y, dy, dy.ptr + 32, ds, *sh), "only g == dy"),
        (lambda: gate(x, y, dy, g, g, *sh), "only g == dy"),
        (lambda: gate(x, y, dy, g, ds, *sh, dy2=dy), "only g == dy"),
        (lambda: gate(x, y, dy, g, ds, N, 46341, 46341, 1), "32-bit index range"),
        (lambda: inp(g, s, dx, 0, H, W, C), "pcnn_se_scale_nhwc_bf16_bwd_input: N = 0"),
        (lambda: inp(g, s, dx, *sh, dpool=dp, dpool_row_pitch=12), "row_pitch 12: 0 \\(C rounded up to 8\\) or a multiple of 8"),
        (lambda: inp(g, s, dx, *sh, dpool=dp, dpool_row_pitch=8), "row_pitch 8"),
        (lambda: inp(None, s, dx, *sh), "NULL context, g, s or dx"),
        (lambda: inp(g, s, None, *sh), "NULL context, g, s or dx"),
        (lambda: inp(g, s.ptr + 2, dx, *sh), "g, s, dpool and dx must be 16-byte aligned"),
        (lambda: inp(g, s, dx, *sh, dpool=dp.ptr + 8), "16-byte aligned"),
        (lambda: inp(g, s, s, *sh), "only dx == g \\(in place\\) may share memory"),
        (lambda: inp(g, s, dx, *sh, dpool=dx), "only dx == g"),
        (lambda: inp(g, s, g.ptr + 16, *sh), "only dx == g"),
        (lambda: inp(g, s, dx, N, 46341, 46341, 1), "32-bit index range"),
    ]
    for fn, msg in cases:
        with pytest.raises(pkg.PcnnError, match=msg):
            fn()
    fwd(x, s, y, *sh, act=3)
    gate(x, y, dy, dy, ds, *sh, act=3)
    inp(dy, s, dy, *sh, dpool=dp, dpool_row_pitch=24)
    eng.sync()


def se_params(rng, C, hid):
    u = lambda shape, fan: rng.uniform(-1, 1, shape).astype(np.float32) / np.float32(np.sqrt(fan))
    return u((hid, C), C), u(hid, C), u((C, hid), hid), u(C, hid)


def lin_bound(x, dy, dw, db):
    """fp32 wgrad / bias sums against float64 on the device's operands: |d - ref| <= 2 n 2^-24 sum |terms| (LinearLayer's bound)"""
    x, dy = x.astype(np.float64), dy.astype(np.float64)
    n = x.shape[0]
    ref_w, ref_b = dy.T @ x, dy.sum(0)
    bw = 2 * n * 2.0 ** -24 * (np.abs(dy).T @ np.abs(x)) + 1e-30
    bb = 2 * n * 2.0 ** -24 * np.abs(dy).sum(0) + 1e-30
    rw, rb = np.abs(dw.reshape(ref_w.shape) - ref_w) / bw, np.abs(db - ref_b) / bb
    return float(max(rw.max(), rb.max()))


def check_layer(pkg, B, L, x, y, r, dy, dy2, g, dx, ds_gate):
    """one SqueezeExcitationLayer forward and backward on its own operands (host bits of x, y, r, dy, dy2, g = dr, dx and the ds
    of a gate pass run on the same operands): y, g, ds and dx bit-exact, fc2's sigmoid gradient bit-exact, the fc dw / db within
    LinearLayer's bound.  Returns the worst ratio to that bound and whether a dx without dpool would have been caught."""
    bits, val = pkg.f32_to_bf16_bits, pkg.bf16_bits_to_f32
    N, H, W, C = L.shape
    rd = lambda d, shape: B.read_plain(d, shape)
    s, a, h, dh = rd(L.s, (N, C)), rd(L.a, (N, L.hidden)), rd(L.h, (N, L.row_pitch)), rd(L.dh, (N, L.row_pitch))
    dpre2, dpre1 = rd(L.ds, (N, C)), rd(L.da, (N, L.hidden))
    assert same_or_nan(y, bits(SR.fwd(val(x), val(s), None if r is None else val(r), L.act))), "y"
    want_g = bits(SR.gate_g(val(dy), val(y), None if dy2 is None else val(dy2), L.act))
    assert np.array_equal(g, want_g), "g"
    want_ds = bits(SR.gate_ds(val(g), val(x), L.info))
    assert np.array_equal(ds_gate, want_ds), "ds"
    assert np.array_equal(dpre2, bits(SR.sigmoid_bwd(val(want_ds), val(s)))), "fc2 dpre"
    want_dx = bits(SR.dx(val(g), val(s), val(dh[:, :C]), H * W))
    assert np.array_equal(dx, want_dx), "dx"
    caught = not np.array_equal(dx, bits(SR.dx(val(g), val(s))))
    w1g, b1g = L.fc1.dw.to_host(), L.fc1.db.to_host()
    w2g, b2g = L.fc2.dw.to_host(), L.fc2.db.to_host()
    ratio = max(lin_bound(val(h[:, :C]), val(dpre1), w1g, b1g), lin_bound(val(a), val(dpre2), w2g, b2g))
    assert ratio <= 1.0, ratio
    return ratio, caught


class Plain(Bufs):
    def read_plain(self, d, shape):
        self.eng.sync()
        return d.to_host().reshape(-1)[:int(np.prod(shape))].reshape(shape)


@pytest.mark.parametrize("act", [0, 3])
def test_layer_step(eng, pkg, act):
    N, H, W, C, hid = 16, 7, 7, 32, 8
    rng = np.random.default_rng(40 + act)
    bits = pkg.f32_to_bf16_bits
    B = Plain(eng)
    L = pkg.SqueezeExcitationLayer(eng, N, H, W, C, hid, *se_params(rng, C, hid), act=act)
    shape, n = (N, H, W, C), N * H * W * C
    try:
        x, r, dy, dy2 = (bits(rng.standard_normal(shape).astype(np.float32)) for _ in range(4))
        x_, r_, dy_, dy2_ = (B.put(a) for a in (x, r, dy, dy2))
        y_, g_, dx_ = B.out(n), B.out(n), B.out(n)
        L.forward(x_, y_, r=r_)
        g_chk, ds_chk = B.out(n), B.out(N * C)
        eng.se_scale_bwd_gate(x_, y_, dy_, g_chk, ds_chk, N, H, W, C, dy2=dy2_, act=act)
        L.backward(y_, dy_, dx_, dr=g_, dy2=dy2_)
        ratio, caught = check_layer(pkg, B, L, x, B.read(y_, shape), r, dy, dy2, B.read(g_, shape), B.read(dx_, shape), B.read(ds_chk, (N, C)))
        assert np.array_equal(B.read(dy_, shape), dy)                                   # with dr, dy is left alone
        assert caught, "a dx without the squeeze branch's gradient would pass"
        # without dr, dy is consumed: g is written over it, and dx may be dy
        L.forward(x_, y_, r=r_)
        L.backward(y_, dy_, dy_, dy2=dy2_)
        assert np.array_equal(B.read(dy_, shape), B.read(dx_, shape))
        print(f"SE layer act {act}: fc dw/db worst ratio to LinearLayer's bound {ratio:.3g}")
    finally:
        L.close()


@pytest.mark.parametrize("kind", ["sgd", "adamw"])
def test_optimizers(eng, pkg, kind):
    """pkg.SGD (momentum, decay) and pkg.AdamW over the layer's four tensors, bit-identical to the float32 replays over 3 steps;
    the layer's forward after a step uses the refreshed plans (the gate equals a fresh layer's on the new masters)"""
    N, H, W, C, hid = 8, 5, 5, 16, 8
    rng = np.random.default_rng(7)
    bits = pkg.f32_to_bf16_bits
    B = Plain(eng)
    L = pkg.SqueezeExcitationLayer(eng, N, H, W, C, hid, *se_params(rng, C, hid), act=3)
    shape, n = (N, H, W, C), N * H * W * C
    x_, dy_ = (B.put(bits(rng.standard_normal(shape).astype(np.float32))) for _ in range(2))
    y_, dx_, g_ = B.out(n), B.out(n), B.out(n)
    opt = pkg.SGD(eng, [L], momentum=0.9, weight_decay=1e-2) if kind == "sgd" else pkg.AdamW(eng, [L], weight_decay=1e-2)
    tensors = L.optim_tensors()
    state = [[None, np.zeros(t[0].nbytes // 4, np.float32), np.zeros(t[0].nbytes // 4, np.float32)] for t in tensors]
    try:
        for t in range(1, 4):
            lr = 0.05 * t
            L.forward(x_, y_)
            L.backward(y_, dy_, dx_, dr=g_)
            eng.sync()
            ps, gs = [p.to_host().reshape(-1) for p, *_ in tensors], [g.to_host().reshape(-1) for _, g, *_ in tensors]
            opt.step(lr)
            eng.sync()
            for i, (p, g) in enumerate(zip(ps, gs)):
                if kind == "sgd":
                    want, state[i][0] = OR.sgd32(p, g, state[i][0], lr, t, momentum=0.9, wd=1e-2)
                else:
                    want, state[i][1], state[i][2] = OR.adamw32(p, g, state[i][1], state[i][2], lr, t, wd=1e-2)
                assert np.array_equal(tensors[i][0].to_host().reshape(-1).view(np.uint32), want.view(np.uint32)), (kind, t, i)
        L.forward(x_, y_)
        s_after = B.read_plain(L.s, (N, C))
        w1, b1, w2, b2 = L.params()
        F = pkg.SqueezeExcitationLayer(eng, N, H, W, C, hid, w1, b1, w2, b2, act=3)
        F.forward(x_, B.out(n))
        assert np.array_equal(B.read_plain(F.s, (N, C)), s_after)
        F.close()
    finally:
        opt.close()
        L.close()


# ------------------------------------------------------------------------------------------------ end to end
ACC_MIN = 0.90          # the float32 torch CPU replica (scripts/seresnet_replica.py) of this network reaches 0.961 (DESIGN 3.19)


def test_seresnet_mnist(eng, pkg, golden):
    """In each of the first 5 steps both SE layers' y, g, dx and fc2 sigmoid gradient are bit-exact against the replays on the
    device's own tensors (ds through that gradient).  A fresh run reproduces the parameters after 5 steps bit for bit.  After
    EPOCHS epochs over the 1024 training digits the mean loss has fallen, and test accuracy on the 256 test digits, evaluated with
    the running statistics, exceeds ACC_MIN."""
    bits, val = pkg.f32_to_bf16_bits, pkg.bf16_bits_to_f32
    B = Plain(eng)
    NB = SEResNet.NB

    def check_step(net, it, x, labels):
        net.forward(x, labels)
        eng.sync()
        fwd = {1: (host(net.z4), host(net.x0), host(net.x1)), 2: (host(net.z6), host(net.s), host(net.out))}
        ss = {1: B.read_plain(net.se1.s, (NB, 16)), 2: B.read_plain(net.se2.s, (NB, 32))}
        net.backward()
        eng.sync()
        for k, L, dy, dy2, g, dx in ((1, net.se1, net.dx1, net.dx1p, net.dres, net.dz4), (2, net.se2, net.dout, None, net.ds, net.dz6)):
            N, H, W, C = L.shape
            x, r, y = fwd[k]
            s = ss[k]
            assert np.array_equal(y, bits(SR.fwd(val(x), val(s), val(r), 3))), (it, k, "y")
            gg, dyh = host(g), host(dy)
            want_g = SR.gate_g(val(dyh), val(y), None if dy2 is None else val(host(dy2)), 3)
            assert np.array_equal(gg, bits(want_g)), (it, k, "g")
            want_ds = bits(SR.gate_ds(val(gg), val(x), L.info))
            assert np.array_equal(B.read_plain(L.ds, (N, C)), bits(SR.sigmoid_bwd(val(want_ds), val(s)))), (it, k, "fc2 dpre")
            dh = B.read_plain(L.dh, (N, L.row_pitch))[:, :C]
            assert np.array_equal(host(dx), bits(SR.dx(val(gg), val(s), val(dh), H * W))), (it, k, "dx")

    ep_loss, acc, _ = train(eng, pkg, golden, lambda: SEResNet(eng, pkg, SEResNet.init_params()), SEResNet.EPOCHS, check_step=check_step)
    print(f"SE-ResNet: mean loss by epoch {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}; test accuracy {acc:.4f} (threshold {ACC_MIN})")
    assert np.isfinite(ep_loss).all() and ep_loss[-1] < ep_loss[0]
    assert acc > ACC_MIN
