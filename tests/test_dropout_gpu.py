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
from example_nets import DEV, NAN_BF16, EfficientNetDropout, host, train

pytestmark = pytest.mark.gpu

SENTINEL = 0x7E57
SEED = 0x0123456789ABCDEF
SPECIAL = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-40, -1e-40, 9.2e-41, -3.0e-39, 3.0e38, -3.0e38, 1.0, -1.0], np.float32)

SHAPES = {  # name: (N, row_elems, row_pitch)
    "nhwc-56x56x64": (128, 56 * 56 * 64, 0), "nhwc-7x7x1280": (128, 7 * 7 * 1280, 0), "gap-C12-pitch16": (128, 12, 16),
    "gap-C1280": (128, 1280, 1280), "odd-7x7x3": (33, 147, 0), "N1-odd": (1, 1001, 0), "N1-vec": (1, 4096, 4104)}
PS = [0.0, 0.1, 0.5, 0.9]


def same_or_nan(got, want):
    """bf16 bits: identical where want is a number; NaN (any payload) where want is NaN"""
    got, want = np.asarray(got, np.uint16), np.asarray(want, np.uint16)
    nan, gnan = (want & 0x7FFF) > 0x7F80, (got & 0x7FFF) > 0x7F80
    return np.array_equal(gnan, nan) and np.array_equal(got[~nan], want[~nan])


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
ACC_MIN = 0.85          # the float32 torch CPU replica (scripts/efficientnet_dropout_replica.py) reaches 0.8945 (DESIGN 3.22)
NB, EPOCHS = EfficientNetDropout.NB, EfficientNetDropout.EPOCHS
P_FC, P_PATH, SEED_FC, SEED_PATH = EfficientNetDropout.P_FC, EfficientNetDropout.P_PATH, EfficientNetDropout.SEED_FC, EfficientNetDropout.SEED_PATH


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
    dropped = 0

    def check_step(net, it, x, labels):
        nonlocal dropped
        net.trace = True
        net.forward(x, labels)
        net.backward()
        eng.sync()
        check_net_dropout(pkg, net)
        dropped += int((~mask(NB, 1, P_PATH, SEED_PATH, it + 1, True)).sum())
        if it == 4:
            assert dropped > 0                      # some image's residual branch was dropped

    def check_trained(net):
        """after training and again after eval, which draws no mask"""
        assert net.drop_fc.call == net.drop_path.call == EPOCHS * 8

    ep_loss, acc, _ = train(eng, pkg, golden, lambda: EfficientNetDropout(eng, pkg, EfficientNetDropout.init_params()), EPOCHS,
                            check_step=check_step, check_trained=check_trained)
    print(f"EfficientNet-style network with dropout and stochastic depth: mean loss by epoch {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}; "
          f"test accuracy {acc:.4f} (threshold {ACC_MIN})")
    assert np.isfinite(ep_loss).all() and ep_loss[-1] < ep_loss[0]
    assert acc > ACC_MIN
