"""Dropout and stochastic depth on the device (pcnn_dropout_bf16, DropoutLayer): y bit for bit against the numpy replay of
dropout_ref.py on dense NHWC activations, global-average-pool rows with and without pad, odd rows (the scalar path) and N = 1, in
both modes, with and without r, at p from 0 to 0.9, with NaN, infinities, both zeros and subnormals in x and r; pad sentinels,
in-place calls, reruns, other calls and seeds, row prefixes and the backward's zeros; the layer in eval; refusals; and an
EfficientNet-style network trained with dropout before its classifier and stochastic depth on its residual block."""
import functools

import numpy as np
import pytest
import torch

import dropout_ref as D
from test_bnact_gpu import DEV, NAN_BF16, NB, EPOCHS, LR_STEP, EfficientNetLite, host, init_params, mnist_device, same_or_nan

pytestmark = pytest.mark.gpu

SENTINEL = 0x7E57
SEED = 0x0123456789ABCDEF
SPECIAL = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-40, -1e-40, 9.2e-41, -3.0e-39, 3.0e38, -3.0e38, 1.0, -1.0], np.float32)

SHAPES = {  # name: (N, row_elems, row_pitch)
    "nhwc-56x56x64": (128, 56 * 56 * 64, 0), "nhwc-7x7x1280": (128, 7 * 7 * 1280, 0), "gap-C12-pitch16": (128, 12, 16),
    "gap-C1280": (128, 1280, 1280), "odd-7x7x3": (33, 147, 0), "N1-odd": (1, 1001, 0), "N1-vec": (1, 4096, 4104)}
PS = [0.0, 0.1, 0.5, 0.9]


@functools.lru_cache(maxsize=None)
def operand(pkg, name, which):
    """(bits [N][pitch] with NaN in the pad, float32 values [N][row_elems]) of a shape: normals with SPECIAL at every 37th element"""
    N, E, pitch = SHAPES[name]
    pitch = pitch or E
    rng = np.random.default_rng([which, *name.encode()])
    v = (rng.standard_normal((N, E)) * 3).astype(np.float32)
    flat = v.reshape(-1)
    idx = np.arange(which, flat.size, 37)
    flat[idx] = SPECIAL[np.arange(idx.size) % SPECIAL.size]
    bits = pkg.f32_to_bf16_bits(v)
    full = np.full((N, pitch), NAN_BF16, np.uint16)
    full[:, :E] = bits
    return full, pkg.bf16_bits_to_f32(bits)


@functools.lru_cache(maxsize=None)
def mask(N, E, p, seed, call, per_sample):
    return D.keep(N, E, p, seed, call, per_sample)


def dev(bits):
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).to(DEV)


def out_buffer(N, E, pitch):
    return torch.full((N, pitch or E), SENTINEL, dtype=torch.int16, device=DEV)


def want_bits(pkg, x, p, call, per_sample, r=None, seed=SEED):
    N, E = x.shape
    return pkg.f32_to_bf16_bits(D.values(x, mask(N, E, p, seed, call, bool(per_sample)), D.threshold(p)[1], r))


def check(got, want, E, pitch):
    got = host(got)
    assert same_or_nan(got[:, :E], want)
    if pitch and pitch > E:
        assert (got[:, E:] == SENTINEL).all()


@pytest.mark.parametrize("with_r", [False, True], ids=["no-r", "r"])
@pytest.mark.parametrize("per_sample", [0, 1], ids=["element", "sample"])
@pytest.mark.parametrize("p", PS)
@pytest.mark.parametrize("name", list(SHAPES))
def test_replay(eng, pkg, name, p, per_sample, with_r):
    N, E, pitch = SHAPES[name]
    xb, x = operand(pkg, name, 0)
    rb, r = operand(pkg, name, 5) if with_r else (None, None)
    xd, rd, yd = dev(xb), dev(rb) if with_r else None, out_buffer(N, E, pitch)
    call = 3
    eng.dropout(xd, yd, N, E, p, SEED, call, per_sample, r=rd, row_pitch=pitch)
    check(yd, want_bits(pkg, x, p, call, per_sample, r), E, pitch)
    info = pkg.dropout_info(N, E, pitch, p, per_sample)
    assert info["vec"] == (8 if E % 8 == 0 and (pitch or E) % 8 == 0 else 1)
    if p > 0 and N * E > 1000:
        kept = mask(N, E, p, SEED, call, bool(per_sample))
        rows = N if per_sample else N * E
        assert abs(kept.mean() - (1 - p)) < 5 * np.sqrt(p * (1 - p) / rows) + 1e-12


@pytest.mark.parametrize("name", ["nhwc-7x7x1280", "gap-C12-pitch16", "odd-7x7x3"])
@pytest.mark.parametrize("per_sample", [0, 1], ids=["element", "sample"])
def test_layout_and_reuse(eng, pkg, name, per_sample):
    """in place (y = x, y = r) gives the out-of-place bits; a rerun repeats them; another call or seed changes them; the first N
    rows of a 2N-row call are the N-row call"""
    N, E, pitch = SHAPES[name]
    p = 0.5
    xb, x = operand(pkg, name, 0)
    rb, r = operand(pkg, name, 5)
    ref = out_buffer(N, E, pitch)
    eng.dropout(dev(xb), ref, N, E, p, SEED, 7, per_sample, r=dev(rb), row_pitch=pitch)
    for target in ("x", "r"):
        xd, rd = dev(xb), dev(rb)
        yd = xd if target == "x" else rd
        eng.dropout(xd, yd, N, E, p, SEED, 7, per_sample, r=rd, row_pitch=pitch)
        assert torch.equal(yd[:, :E], ref[:, :E]), target
    again = out_buffer(N, E, pitch)
    eng.dropout(dev(xb), again, N, E, p, SEED, 7, per_sample, r=dev(rb), row_pitch=pitch)
    assert torch.equal(again, ref)
    for seed, call in ((SEED, 8), (SEED + 1, 7), (SEED + (1 << 32), 7), (SEED, 7 + (1 << 32))):
        other = out_buffer(N, E, pitch)
        eng.dropout(dev(xb), other, N, E, p, seed, call, per_sample, r=dev(rb), row_pitch=pitch)
        assert not torch.equal(other, ref), (seed, call)
        check(other, want_bits(pkg, x, p, call, per_sample, r, seed=seed), E, pitch)
    x2 = np.concatenate([xb, xb[::-1]])
    y2 = out_buffer(2 * N, E, pitch)
    eng.dropout(dev(x2), y2, 2 * N, E, p, SEED, 7, per_sample, row_pitch=pitch)
    y1 = out_buffer(N, E, pitch)
    eng.dropout(dev(xb), y1, N, E, p, SEED, 7, per_sample, row_pitch=pitch)
    assert torch.equal(y2[:N], y1)


@pytest.mark.parametrize("per_sample", [0, 1], ids=["element", "sample"])
def test_backward_zero_where_dropped(eng, pkg, per_sample):
    """the backward, the same call on dy, is zero exactly where the forward dropped and dy * scale elsewhere"""
    N, E = 128, 14 * 14 * 112
    rng = np.random.default_rng(4)
    nz = lambda: pkg.f32_to_bf16_bits((rng.uniform(0.5, 2, (N, E)) * rng.choice([-1, 1], (N, E))).astype(np.float32))
    xb, dyb = nz(), nz()
    y, dx = out_buffer(N, E, 0), out_buffer(N, E, 0)
    layer = pkg.DropoutLayer(eng, N, E, 0.2, seed=99, per_sample=bool(per_sample))
    layer.forward(dev(xb), y)
    layer.forward(dev(xb), y)                      # the backward takes the most recent call
    assert layer.call == 2
    dyd = dev(dyb)
    layer.backward(dyd, dx)
    dropped = (host(y) & 0x7FFF) == 0               # +0, or -0 for a negative x
    assert (dropped == ((host(dx) & 0x7FFF) == 0)).all()
    assert np.array_equal(dropped, ~mask(N, E, 0.2, 99, 2, bool(per_sample)))
    assert np.array_equal(host(dx), want_bits(pkg, pkg.bf16_bits_to_f32(dyb), 0.2, 2, per_sample, seed=99))
    layer.backward(dyd, dyd)                        # in place
    assert torch.equal(dyd, dx)


def test_layer_eval(eng, pkg):
    """eval is the p = 0 path: y = x, or x + r; nothing is launched when y is x and there is no r"""
    name = "gap-C12-pitch16"
    N, E, pitch = SHAPES[name]
    xb, x = operand(pkg, name, 0)
    rb, r = operand(pkg, name, 5)
    layer = pkg.DropoutLayer(eng, N, E, 0.5, seed=1, row_pitch=pitch)
    xd, y = dev(xb), out_buffer(N, E, pitch)
    layer.forward(xd, y, training=False)
    check(y, pkg.f32_to_bf16_bits(x), E, pitch)
    layer.forward(xd, y, r=dev(rb), training=False)
    check(y, pkg.f32_to_bf16_bits(D.values(x, np.ones(x.shape, bool), 1.0, r)), E, pitch)
    eng.sync()
    n0 = eng.launch_count()
    layer.forward(xd, xd, training=False)
    assert eng.launch_count() == n0 and layer.call == 0
    assert torch.equal(xd, dev(xb))


def test_refusals(eng, pkg):
    x, y = out_buffer(4, 64, 0), out_buffer(4, 64, 0)
    cases = [(dict(x=None), "NULL context, x or y"), (dict(y=None), "NULL context, x or y"),
             (dict(x=x.data_ptr() + 2), "16-byte aligned"), (dict(r=y.data_ptr() + 16), "16-byte aligned|overlapping"),
             (dict(y=x.data_ptr() + 16), "overlapping buffers"), (dict(p=1.0), "0 <= p < 1"), (dict(N=0), "each must be >= 1"),
             (dict(pitch=32), "row_pitch = 32"), (dict(ps=3), "per_sample = 3")]
    for kw, msg in cases:
        a = dict(x=x, y=y, r=None, N=4, p=0.1, pitch=0, ps=0)
        a.update(kw)
        with pytest.raises(pkg.PcnnError, match=msg):
            eng.dropout(a["x"], a["y"], a["N"], 64, a["p"], 1, 1, a["ps"], r=a["r"], row_pitch=a["pitch"])
    eng.dropout(x, x, 4, 64, 0.1, 1, 1, r=x)      # the same buffer three times is allowed


# ------------------------------------------------------------------------------------------------ end to end
P_FC, P_PATH = 0.2, 0.2
SEED_FC, SEED_PATH = 1001, 2002
ACC_MIN = 0.85          # the float32 torch CPU replica (scripts/efficientnet_dropout_replica.py) reaches 0.8945 (DESIGN 3.22)


class EfficientNetDropout(EfficientNetLite):
    """test_bnact_gpu's EfficientNet-style network with both regularisers: element dropout (p = 0.2) in place on the global
    average pool's output before the fc, and stochastic depth (p = 0.2, per image) on the residual MBConv, whose last BN runs
    without r while the DropoutLayer adds x1.  With `trace` the layers' inputs that the in-place calls overwrite are kept."""

    def __init__(self, eng, pkg, p):
        super().__init__(eng, pkg, p)
        self.drop_fc = pkg.DropoutLayer(eng, NB, 128, P_FC, SEED_FC, row_pitch=self.gap.row_pitch)
        self.drop_path = pkg.DropoutLayer(eng, NB, 6 * 6 * 48, P_PATH, SEED_PATH, per_sample=True)
        self.b2, self.db2 = (torch.full((NB, 6, 6, 48), NAN_BF16, dtype=torch.int16, device=DEV) for _ in range(2))
        self.trace = False

    def snapshot(self, t):
        """a copy of t as the engine's stream has written it, taken before the engine's next call overwrites it (torch copies on
        its own stream)"""
        self.eng.sync()
        copy = t.clone()
        torch.cuda.synchronize()
        return copy

    def forward(self, x, labels, training=True):
        b0, be1, bd1, bp1, be2, bd2, bp2, bh = self.bn
        self.stem.forward(x, self.y0)
        b0.forward(self.y0, self.z0, training=training)
        self.pool.forward(self.z0, self.x1p)
        self.e1.forward(self.x1p, self.ye1)
        be1.forward(self.ye1, self.ze1, training=training)
        self.d1.forward(self.ze1, self.yd1)
        bd1.forward(self.yd1, self.zd1, training=training)
        self.p1.forward(self.zd1, self.yp1)
        bp1.forward(self.yp1, self.x1, training=training)
        self.e2.forward(self.x1, self.ye2)
        be2.forward(self.ye2, self.ze2, training=training)
        self.d2.forward(self.ze2, self.yd2)
        bd2.forward(self.yd2, self.zd2, training=training)
        self.se.forward(self.zd2, self.se_y)
        self.p2.forward(self.se_y, self.yp2)
        bp2.forward(self.yp2, self.b2, training=training)                          # the branch's last BN, without r
        self.drop_path.forward(self.b2, self.x2, r=self.x1, training=training)       # x2 = x1 + drop_path(b2)
        self.hd.forward(self.x2, self.yh)
        bh.forward(self.yh, self.zh, training=training)
        self.gap.forward(self.zh, self.hp)
        if self.trace:
            self.hp_in = self.snapshot(self.hp)
        self.drop_fc.forward(self.hp, self.hp, training=training)
        self.fc.forward(self.hp, self.z)
        self.eng.softmax_ce_bf16(self.z, labels, NB, 10, 1.0 / NB, self.dz, self.loss, self.pred)

    def backward(self):
        b0, be1, bd1, bp1, be2, bd2, bp2, bh = self.bn
        self.fc.backward(self.z, self.dz, self.dhp)
        if self.trace:
            self.dhp_in = self.snapshot(self.dhp)
        self.drop_fc.backward(self.dhp, self.dhp)
        self.gap.backward(self.dhp, self.dzh)
        bh.backward(self.zh, self.dzh, self.dyh, dr=self.gh)
        self.hd.backward(self.yh, self.dyh, self.dx2)
        self.drop_path.backward(self.dx2, self.db2)                                  # dx2 still feeds the skip path
        bp2.backward(self.b2, self.db2, self.dyp2)
        self.p2.backward(self.yp2, self.dyp2, self.dse_y)
        self.se.backward(self.se_y, self.dse_y, self.dzd2)
        bd2.backward(self.zd2, self.dzd2, self.dyd2, dr=self.gd2)
        self.d2.backward(self.yd2, self.dyd2, self.dze2)
        be2.backward(self.ze2, self.dze2, self.dye2, dr=self.ge2)
        self.e2.backward(self.ye2, self.dye2, self.dx1b)
        bp1.backward(self.x1, self.dx1b, self.dyp1, dy2=self.dx2)                   # the block's two paths meet at x1
        self.p1.backward(self.yp1, self.dyp1, self.dzd1)
        bd1.backward(self.zd1, self.dzd1, self.dyd1, dr=self.gd1)
        self.d1.backward(self.yd1, self.dyd1, self.dze1)
        be1.backward(self.ze1, self.dze1, self.dye1, dr=self.ge1)
        self.e1.backward(self.ye1, self.dye1, self.dx1p)
        self.pool.backward(self.dx1p, self.dz0)
        b0.backward(self.z0, self.dz0, self.dy0, dr=self.g0)
        self.stem.backward(self.y0, self.dy0, None)

    def close(self):
        super().close()
        self.drop_fc.close()
        self.drop_path.close()


def check_net_dropout(pkg, net):
    """both layers' outputs and input gradients of the last step against the replay on the device's own operands"""
    f32 = lambda t, E: pkg.bf16_bits_to_f32(host(t).reshape(NB, -1)[:, :E])
    c = net.drop_fc.call
    pitch = net.gap.row_pitch
    want = want_bits(pkg, f32(net.hp_in, 128), P_FC, c, 0, seed=SEED_FC)
    assert same_or_nan(host(net.hp).reshape(NB, pitch)[:, :128], want), ("fc dropout y", c)
    want = want_bits(pkg, f32(net.dhp_in, 128), P_FC, c, 0, seed=SEED_FC)
    assert same_or_nan(host(net.dhp).reshape(NB, pitch)[:, :128], want), ("fc dropout dx", c)
    E = 6 * 6 * 48
    c = net.drop_path.call
    want = want_bits(pkg, f32(net.b2, E), P_PATH, c, 1, r=f32(net.x1, E), seed=SEED_PATH)
    assert same_or_nan(host(net.x2).reshape(NB, E), want), ("drop path y", c)
    want = want_bits(pkg, f32(net.dx2, E), P_PATH, c, 1, seed=SEED_PATH)
    assert same_or_nan(host(net.db2).reshape(NB, E), want), ("drop path dx", c)


def test_efficientnet_dropout_mnist(eng, pkg, golden):
    """In each of the first 5 steps both dropout layers' y and dx are bit-exact against the replay on the device's own operands.
    A second fresh run with the same seeds reproduces the parameters after 5 steps bit for bit.  After EPOCHS epochs over the 1024
    training digits the mean loss has fallen, and test accuracy on the 256 test digits, evaluated with the running statistics and
    without dropout, exceeds ACC_MIN."""
    xs, ys = mnist_device(pkg, golden["train_u8"]), torch.from_numpy(golden["train_labels"]).to(DEV)
    xt, yt = mnist_device(pkg, golden["test_u8"]), torch.from_numpy(golden["test_labels"]).to(DEV)
    row_bytes = 28 * 32 * 2
    batch = lambda s, xs=xs, ys=ys: (xs.data_ptr() + s * NB * row_bytes, ys[s * NB:(s + 1) * NB])

    net = EfficientNetDropout(eng, pkg, init_params())
    net.trace = True
    try:
        dropped = 0
        for it in range(5):
            net.forward(*batch(it))
            net.backward()
            eng.sync()
            check_net_dropout(pkg, net)
            dropped += int((~mask(NB, 1, P_PATH, SEED_PATH, it + 1, True)).sum())
            net.sgd(LR_STEP)
            eng.sync()
        assert dropped > 0                          # some image's residual branch was dropped
        after5 = net.params()
    finally:
        net.close()

    net = EfficientNetDropout(eng, pkg, init_params())
    try:
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
        assert net.drop_fc.call == net.drop_path.call == EPOCHS * 8
        ep_loss = [float(torch.stack(losses[e * 8:(e + 1) * 8]).double().mean()) for e in range(EPOCHS)]
        right = 0
        for s in range(2):
            net.forward(*batch(s, xt, yt), training=False)
            eng.sync()
            right += int((net.pred.cpu().numpy() == golden["test_labels"][s * NB:(s + 1) * NB]).sum())
        assert net.drop_fc.call == EPOCHS * 8
        acc = right / 256
    finally:
        net.close()
    print(f"EfficientNet-style network with dropout and stochastic depth: mean loss by epoch {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}; "
          f"test accuracy {acc:.4f} (threshold {ACC_MIN})")
    assert np.isfinite(ep_loss).all() and ep_loss[-1] < ep_loss[0]
    assert acc > ACC_MIN
