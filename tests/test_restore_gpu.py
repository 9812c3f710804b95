"""Image-to-image regression on the H100: pixel shuffle and unshuffle (pcnn_pixel_shuffle_nhwc_bf16 / pcnn_pixel_unshuffle_nhwc_bf16,
PixelShuffleLayer, PixelUnshuffleLayer) and the regression losses (pcnn_regression_loss_bf16) bit for bit against restore_ref.py,
parity with torch's CUDA autograd, the refusals, and both layers inside SGD and AdamW steps of a small network."""
import numpy as np
import pytest
import torch

import restore_ref as RR
from example_nets import DEV, host, nan_buf

pytestmark = pytest.mark.gpu
NAN = 0x7FC0
TAIL = 64
F = torch.nn.functional


def dev_bits(bits):
    return torch.from_numpy(np.ascontiguousarray(bits, np.uint16).view(np.int16)).to(DEV)


def random_bits(rng, shape):
    """bf16 bits of every kind: normal values, NaNs with payloads of both signs, +-Inf, +-0 and subnormals"""
    b = rng.integers(0, 1 << 16, shape, dtype=np.uint32).astype(np.uint16)
    flat = b.reshape(-1)
    flat[:8] = [0x7F80, 0xFF80, 0x0000, 0x8000, 0x7FC1, 0xFFAB, 0x0001, 0x8003][:flat.size]
    return b


def run_op(eng, fn, xb, out_elems):
    """fn(x, y) on a device copy of xb into a NaN-filled buffer of out_elems + TAIL: (y bits, canaries intact)"""
    y = nan_buf(out_elems + TAIL)
    fn(dev_bits(xb), y)
    eng.sync()
    yb = host(y)
    return yb[:out_elems], bool(np.all(yb[out_elems:] == NAN))


SHUFFLE = [  # N, H, W, C (fine channels), r: every r, C % 8 zero and not, N 1 .. 128, and the benchmark shapes' coarse sides
    (1, 1, 1, 1, 1), (2, 5, 7, 3, 1), (1, 3, 4, 1, 2), (2, 7, 5, 3, 2), (3, 4, 6, 8, 2), (1, 5, 3, 24, 3), (2, 3, 3, 5, 4),
    (1, 2, 3, 16, 5), (1, 2, 2, 7, 6), (1, 3, 2, 32, 7), (2, 2, 3, 9, 8), (1, 2, 2, 64, 8), (1, 3, 2, 256, 4), (4, 6, 5, 256, 2),
    (128, 4, 4, 8, 2), (128, 3, 3, 1, 3), (5, 9, 11, 136, 2), (2, 1, 1, 1000, 5),
    (16, 128, 128, 3, 2), (16, 64, 64, 3, 4), (16, 48, 48, 64, 2), (16, 96, 96, 64, 2), (128, 28, 28, 64, 2),
]


@pytest.mark.parametrize("N,H,W,C,r", SHUFFLE)
def test_shuffle_and_unshuffle_bit_exact(pkg, eng, N, H, W, C, r):
    rng = np.random.default_rng(N * 7 + H * 5 + C * 3 + r)
    x = random_bits(rng, (N, H, W, C * r * r))
    y, ok = run_op(eng, lambda a, b: eng.pixel_shuffle(a, b, N, H, W, C, r), x, x.size)
    want = RR.shuffle(x, r)
    assert ok and np.array_equal(y, want.reshape(-1))
    back, ok = run_op(eng, lambda a, b: eng.pixel_unshuffle(a, b, N, H * r, W * r, C, r), y.reshape(want.shape), x.size)
    assert ok and np.array_equal(back, x.reshape(-1))              # unshuffle(shuffle(x)) == x
    fine = random_bits(rng, (N, H * r, W * r, C))
    u, ok = run_op(eng, lambda a, b: eng.pixel_unshuffle(a, b, N, H * r, W * r, C, r), fine, fine.size)
    assert ok and np.array_equal(u, RR.unshuffle(fine, r).reshape(-1))


@pytest.mark.parametrize("N,H,W,C,r", [(2, 7, 5, 3, 2), (3, 4, 6, 8, 2), (1, 5, 3, 24, 3)])
def test_layers_backward_is_the_other_direction(pkg, eng, N, H, W, C, r):
    rng = np.random.default_rng(C + r)
    ps, pu = pkg.PixelShuffleLayer(eng, N, H, W, C, r), pkg.PixelUnshuffleLayer(eng, N, H * r, W * r, C, r)
    assert ps.out_shape == (N, H * r, W * r, C) and pu.out_shape == (N, H, W, C * r * r)
    assert ps.info == pkg.pixel_shuffle_info(N, H, W, C, r) and pu.info == pkg.pixel_shuffle_info(N, H * r, W * r, C, r, unshuffle=True)
    dy_fine, dy_coarse = random_bits(rng, (N, H * r, W * r, C)), random_bits(rng, (N, H, W, C * r * r))
    a, ok1 = run_op(eng, ps.backward, dy_fine, dy_fine.size)
    b, ok2 = run_op(eng, pu.forward, dy_fine, dy_fine.size)
    c, ok3 = run_op(eng, pu.backward, dy_coarse, dy_coarse.size)
    d, ok4 = run_op(eng, ps.forward, dy_coarse, dy_coarse.size)
    assert ok1 and ok2 and ok3 and ok4 and np.array_equal(a, b) and np.array_equal(c, d)
    assert np.array_equal(a, RR.unshuffle(dy_fine, r).reshape(-1)) and np.array_equal(c, RR.shuffle(dy_coarse, r).reshape(-1))


def loss_operands(rng, P, C, ts, special):
    p = rng.standard_normal((P, C)).astype(np.float32)
    t = rng.standard_normal((P, ts)).astype(np.float32)
    if special:
        pv = [0.0, -0.0, 0.0, np.nan, np.inf, -np.inf, 1.0, 3e38, 2.5]
        tv = [0.0, 0.0, -0.0, 0.0, 1.0, 1.0, np.nan, -3e38, 2.5]
        for k, (a, b) in enumerate(zip(pv, tv)):
            p[k % P, k % C], t[k % P, k % C] = a, b
    return RR.bf16_bits(p), RR.bf16_bits(t)


LOSS = [  # pixels, C, target_stride, special: both paths, pitched targets, more channels than one pass over shared memory
    (1, 1, 1, False), (1000, 1, 8, True), (4097, 3, 3, True), (300, 3, 7, False), (513, 8, 8, True), (200, 16, 24, True),
    (130, 8, 12, False), (77, 64, 64, True), (65, 136, 144, False), (9, 250, 250, True), (64 * 50 + 3, 24, 32, False),
]


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("P,C,ts,special", LOSS)
def test_loss_bit_exact(pkg, eng, mode, P, C, ts, special):
    rng = np.random.default_rng(P + C + ts + mode)
    pb, tb = loss_operands(rng, P, C, ts, special)
    scale = float(rng.uniform(0.1, 2.0)) / (P * C)
    want_g, want_l = RR.loss_replay(pb, tb, C, mode, scale, target_stride=ts)
    pred, target = dev_bits(pb), dev_bits(tb)
    d = nan_buf(P * C + TAIL)
    loss = torch.full((P + 16,), float("nan"), device=DEV)
    eng.regression_loss_bf16(pred, target, P, C, d, loss, mode=mode, target_stride=ts, scale=scale)
    eng.sync()
    db, lh = host(d), loss.cpu().numpy()
    assert np.all(db[P * C:] == NAN) and np.all(np.isnan(lh[P:]))
    assert np.array_equal(db[:P * C], want_g.reshape(-1))
    nanl = np.isnan(want_l)                                         # a NaN loss is any NaN
    assert np.array_equal(np.isnan(lh[:P]), nanl) and np.array_equal(lh[:P][~nanl].view(np.uint32), want_l[~nanl].view(np.uint32))
    # no loss, rerun, in place: the same dpred bits
    d2 = nan_buf(P * C)
    eng.regression_loss_bf16(pred, target, P, C, d2, None, mode=mode, target_stride=ts, scale=scale)
    eng.regression_loss_bf16(pred, target, P, C, pred, None, mode=mode, target_stride=ts, scale=scale)
    eng.sync()
    assert np.array_equal(host(d2), want_g.reshape(-1)) and np.array_equal(host(pred).reshape(-1), want_g.reshape(-1))


def test_loss_default_scale_is_the_mean(pkg, eng):
    rng = np.random.default_rng(3)
    pb, tb = loss_operands(rng, 500, 8, 8, False)
    d = nan_buf(500 * 8)
    eng.regression_loss_bf16(dev_bits(pb), dev_bits(tb), 500, 8, d)
    eng.sync()
    assert np.array_equal(host(d), RR.loss_replay(pb, tb, 8, RR.MSE, 1.0 / 4000)[0].reshape(-1))


def _ulps(a, b):
    """|a - b| in bf16 ulps of the larger magnitude (float32 arrays of bf16 values)"""
    m = np.maximum(np.abs(a), np.abs(b))
    ulp = np.exp2(np.floor(np.log2(np.where(m > 0, m, 1.0))) - 7)
    return np.abs(a - b) / ulp


@pytest.mark.parametrize("mode", [0, 1])
def test_loss_parity_with_torch_cuda_autograd(pkg, eng, mode):
    """On the same bf16 tensors, upcast to float32 and as they are: torch's CUDA autograd is within one bf16 ulp of dpred (in bf16
    torch rounds p - t and 2 / n to bf16 before its product) and its float32 mean loss within fp32 summation error of ours.  Its
    special values are printed beside ours; on an H100 they agree (pcnn.h)."""
    rng = np.random.default_rng(11 + mode)
    P, C = 20000, 3
    pb, tb = loss_operands(rng, P, C, C, False)
    d, loss = nan_buf(P * C), torch.zeros(P, device=DEV)
    eng.regression_loss_bf16(dev_bits(pb), dev_bits(tb), P, C, d, loss, mode=mode)
    eng.sync()
    ours = RR.bits_f32(host(d)).reshape(P, C)
    fn = F.mse_loss if mode == RR.MSE else F.l1_loss
    for dt in (torch.float32, torch.bfloat16):
        pt = dev_bits(pb).view(torch.bfloat16).to(dt).reshape(P, C).requires_grad_(True)
        tt = dev_bits(tb).view(torch.bfloat16).to(dt).reshape(P, C)
        lt = fn(pt, tt)
        lt.backward()
        theirs = pt.grad.float().cpu().numpy()
        worst = float(_ulps(ours, theirs).max())
        print(f"mode {mode} torch {dt}: worst dpred difference {worst} bf16 ulp")
        assert worst <= 1.0
        if dt == torch.float32:
            mean = loss.double().sum().item() / (P * C)
            assert abs(mean - lt.item()) <= 1e-5 * abs(mean)
    sp = np.array([[0.0, -0.0, np.nan, np.inf, -np.inf, 1.0]], np.float32)
    st = np.array([[0.0, 0.0, 0.0, 1.0, 1.0, np.nan]], np.float32)
    pt = torch.from_numpy(sp).to(DEV).requires_grad_(True)
    fn(pt, torch.from_numpy(st).to(DEV)).backward()
    mine = RR.bits_f32(RR.loss_replay(RR.bf16_bits(sp), RR.bf16_bits(st), 6, mode, 1.0 / 6)[0]).reshape(-1)
    print(f"mode {mode} special values: torch CUDA float32 {pt.grad.cpu().numpy().reshape(-1).tolist()}, ours {mine.tolist()}")


def test_refusals(pkg, eng):
    x, y = nan_buf(4096), nan_buf(4096)
    for args, msg in (((x, y, 1, 4, 4, 8, 9), "r = 9"), ((x, y, 1, 4, 4, 0, 2), "C = 0"), ((x, y.data_ptr() + 2, 1, 4, 4, 8, 2), "16-byte"),
                      ((x, x.data_ptr() + 64, 1, 4, 4, 8, 2), "overlap"), ((None, y, 1, 4, 4, 8, 2), "NULL")):
        with pytest.raises(pkg.PcnnError, match=msg):
            eng.pixel_shuffle(*args)
    with pytest.raises(pkg.PcnnError, match="multiples of r"):
        eng.pixel_unshuffle(x, y, 1, 6, 4, 8, 4)
    with pytest.raises(pkg.PcnnError, match="overlap"):
        eng.pixel_unshuffle(x, x, 1, 4, 4, 8, 2)
    loss = torch.zeros(64, device=DEV)
    for kw, msg in ((dict(pixels=0), "pixels = 0"), (dict(C=9, target_stride=8), "target_stride"), (dict(mode=2), "mode 2"),
                    (dict(scale=float("inf")), "finite scale"), (dict(dpred=y.data_ptr() + 2), "16-byte"),
                    (dict(dpred=x.data_ptr() + 16), "only dpred == pred"), (dict(dpred=y, target=y), "dpred overlaps target"),
                    (dict(loss=x), "loss overlaps"), (dict(pred=None), "NULL")):
        a = dict(pred=x, target=nan_buf(1024), pixels=64, C=8, dpred=y, loss=loss, mode=0, target_stride=8, scale=None)
        a.update(kw)
        with pytest.raises(pkg.PcnnError, match=msg):
            eng.regression_loss_bf16(a["pred"], a["target"], a["pixels"], a["C"], a["dpred"], a["loss"], a["mode"], a["target_stride"],
                                     a["scale"])


@pytest.mark.parametrize("opt_name", ["SGD", "AdamW"])
def test_layers_in_an_optimizer_step(pkg, eng, opt_name):
    """x [N][8][8][16] -> unshuffle x2 -> per-pixel fc 64->32 -> shuffle x2 -> [N][8][8][8] -> MSE against a pitched target: every
    shuffle, unshuffle and loss bit against the replays in three steps, and the loss goes down"""
    N, r = 4, 2
    rng = np.random.default_rng(5)
    w = (rng.standard_normal((32, 1, 1, 64)) / 8).astype(np.float32)
    b = np.zeros(32, np.float32)
    un = pkg.PixelUnshuffleLayer(eng, N, 8, 8, 16, r)
    fc = pkg.LinearLayer(eng, N * 16, 1, 1, 64, 32, w, b, row_pitch=64)
    ps = pkg.PixelShuffleLayer(eng, N, 4, 4, 8, r)
    opt = pkg.SGD(eng, [fc], momentum=0.9) if opt_name == "SGD" else pkg.AdamW(eng, [fc])
    xb = RR.bf16_bits(rng.standard_normal((N, 8, 8, 16)).astype(np.float32))
    tb = RR.bf16_bits(rng.standard_normal((N * 64, 16)).astype(np.float32))
    x, target = dev_bits(xb), dev_bits(tb)
    u, z, out, dout, dz, du = nan_buf(N, 4, 4, 64), nan_buf(N * 16, 32), nan_buf(N, 8, 8, 8), nan_buf(N, 8, 8, 8), nan_buf(N * 16, 32), \
        nan_buf(N, 4, 4, 64)
    dx, loss = nan_buf(N, 8, 8, 16), torch.zeros(N * 64, device=DEV)
    means = []
    try:
        for _ in range(3):
            un.forward(x, u)
            fc.forward(u, z)
            ps.forward(z, out)
            eng.regression_loss_bf16(out, target, N * 64, 8, dout, loss, target_stride=16)
            ps.backward(dout, dz)
            fc.backward(z, dz, du)
            un.backward(du, dx)
            eng.sync()
            assert np.array_equal(host(u).reshape(N, 4, 4, 64), RR.unshuffle(xb, r))
            assert np.array_equal(host(out).reshape(N, 8, 8, 8), RR.shuffle(host(z).reshape(N, 4, 4, 32), r))
            g, lw = RR.loss_replay(host(out), tb, 8, RR.MSE, 1.0 / (N * 64 * 8), target_stride=16)
            assert np.array_equal(host(dout).reshape(-1), g.reshape(-1)) and np.array_equal(loss.cpu().numpy().view(np.uint32), lw.view(np.uint32))
            assert np.array_equal(host(dz).reshape(N, 4, 4, 32), RR.unshuffle(host(dout).reshape(N, 8, 8, 8), r))
            assert np.array_equal(host(dx).reshape(N, 8, 8, 16), RR.shuffle(host(du).reshape(N, 4, 4, 64), r))
            means.append(float(lw.astype(np.float64).sum()))
            opt.step(0.05 if opt_name == "SGD" else 0.01)
            eng.sync()
        assert means[2] < means[0]
    finally:
        opt.close()
        fc.close()
