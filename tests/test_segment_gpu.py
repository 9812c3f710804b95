"""Dense prediction on the H100: the transposed convolution (ConvTransposeLayer, pcnn_conv_transpose_fwd), the bilinear resize, the
per-pixel cross-entropy and the mask batch against segment_ref.py, and the two segmenters of segment_nets.py trained end to end."""
import numpy as np
import pytest
import torch

import linear_ref
import segment_ref as SR
from example_nets import DEV, host, nan_buf
import segment_nets

pytestmark = pytest.mark.gpu
NAN = 0x7FC0


def dev_bits(bits):
    return torch.from_numpy(np.ascontiguousarray(bits, np.uint16).view(np.int16)).to(DEV)


def guarded(n, tail=64):
    """a NaN-filled bf16 buffer of n + tail elements: the tail must stay NaN"""
    return nan_buf(n + tail)


def ints(rng, shape, lo=-3, hi=4, density=1.0):
    """small integers, a fraction `density` of them nonzero, so that every sum below stays an integer bf16 holds exactly"""
    return (rng.integers(lo, hi, shape) * (rng.random(shape) < density)).astype(np.float32)


def _f64(pkg, t, shape):
    return pkg.bf16_bits_to_f32(host(t)).reshape(shape).astype(np.float64)


def check_convt(pkg, layer, x, y, dpre=None, dx=None):
    """a ConvTransposeLayer's y (and, given the gradient dpre at the pre-activation that its last backward consumed, its dx and dw)
    on its own bf16 operands and master against segment_ref's float64 passes: y and dx within bf16 rounding plus an fp32
    accumulation bound, dw (fp32) within the fp32 bound of its sum over N H W pixels.  Call it before the optimizer step."""
    N, H, W, Ci, Co, R, S = layer.shape
    _, Ho, Wo, _ = layer.out_shape
    st, pad, op = layer.stride, layer.padding, layer.output_padding
    xq = _f64(pkg, x, (N, H, W, Ci))
    wq = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(layer.weight())).astype(np.float64)
    b = None if layer.bias is None else layer.bias.to_host().astype(np.float64)
    _, want = SR.convt_fwd_f64(xq, wq, b, st, pad, op, layer.act)
    absum = SR.convt_fwd_f64(np.abs(xq), np.abs(wq), None if b is None else np.abs(b), st, pad, op)[0]
    got = _f64(pkg, y, want.shape)
    assert np.all(np.abs(got - want) <= 2 ** -8 * np.abs(want) + 2 ** -18 * absum + 1e-30), "convT y"
    if dpre is None:
        return
    dq = _f64(pkg, dpre, (N, Ho, Wo, Co))
    rdx, rdw, _ = SR.convt_bwd_f64(xq, wq, dq, st, pad)
    adx, adw, _ = SR.convt_bwd_f64(np.abs(xq), np.abs(wq), np.abs(dq), st, pad)
    gdx = _f64(pkg, dx, rdx.shape)
    assert np.all(np.abs(gdx - rdx) <= 2 ** -8 * np.abs(rdx) + 2 ** -18 * adx + 1e-30), "convT dx"
    gdw = layer.dw.to_host().reshape(Ci, R, S, Co).transpose(0, 3, 1, 2).astype(np.float64)
    assert np.all(np.abs(gdw - rdw) <= (N * H * W * 2.0 ** -24 + 2.0 ** -20) * adw + 1e-30), "convT dw"


def dpre_of(pkg, y, dy, act, shape):
    """pcnn_conv_bias_act_bwd's gradient at the pre-activation on host copies of y and dy (bf16 bits): act 0 dy, act 3 dy where
    y > 0 (else +0), act 1 bf16_rn(dy * (y * (1 - y))) in fp32"""
    yb, dyb = host(y).reshape(shape), host(dy).reshape(shape)
    if act == 0:
        return dyb
    yf, dyf = pkg.bf16_bits_to_f32(yb), pkg.bf16_bits_to_f32(dyb)
    if act == 3:
        return np.where(yf <= 0, np.uint16(0), dyb).astype(np.uint16)
    return pkg.f32_to_bf16_bits(dyf * (yf * (np.float32(1) - yf)))


CONVT = [  # N, H, W, C_in, C_out, R, S, stride, padding, output_padding
    (2, 7, 7, 64, 32, 4, 4, 2, (1, 1), (0, 0)),
    (2, 14, 14, 32, 16, 4, 4, 2, (1, 1), (0, 0)),
    (1, 5, 6, 16, 24, 3, 3, 2, (1, 1), (1, 1)),
    (2, 4, 5, 8, 32, 3, 3, 3, (1, 0), (2, 1)),
    (1, 3, 4, 16, 16, 2, 2, 4, (0, 0), (3, 2)),     # stride > taps: pixels no window reaches
    (1, 6, 6, 256, 264, 3, 3, 1, (1, 1), (0, 0)),   # two channel groups
]


def _convt_layer(pkg, eng, shape, w, b=None, act=0):
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    return pkg.ConvTransposeLayer(eng, N, H, W, Ci, Co, R, S, w, b, act=act, stride=st, padding=pad, output_padding=op)


@pytest.mark.parametrize("shape", CONVT)
def test_convt_integer_operands_exact(pkg, eng, shape):
    """y, dx and dw equal the float64 reference bit for bit on small integers; <y, dy> = <x, dx> = <w, dw> exactly"""
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    rng = np.random.default_rng(sum(shape[:8]))
    dens = 0.1 if Ci > 64 else 1.0
    x, w = ints(rng, (N, H, W, Ci), density=dens), ints(rng, (Ci, Co, R, S), -2, 3, dens)
    b = None if Co > 256 else ints(rng, Co)
    layer = _convt_layer(pkg, eng, shape, w, b)
    try:
        _, Ho, Wo, _ = layer.out_shape
        xd = dev_bits(pkg.f32_to_bf16_bits(x))
        y = guarded(N * Ho * Wo * Co)
        layer.forward(xd, y)
        eng.sync()
        yb = host(y)
        assert np.all(yb[-64:] == NAN)
        _, want = SR.convt_fwd_f64(x, w, b, st, pad, op)
        got = pkg.bf16_bits_to_f32(yb[:-64]).reshape(want.shape)
        assert np.abs(want).max() < 256 and np.array_equal(got, want.astype(np.float32))
        dy = ints(rng, want.shape, -2, 3, dens)
        dyd = dev_bits(pkg.f32_to_bf16_bits(dy))
        dx = guarded(N * H * W * Ci)
        layer.backward(y, dyd, dx)
        eng.sync()
        dxb = host(dx)
        assert np.all(dxb[-64:] == NAN)
        rdx, rdw, rdb = SR.convt_bwd_f64(x, w, dy, st, pad)
        gdx = pkg.bf16_bits_to_f32(dxb[:-64]).reshape(rdx.shape)
        assert np.abs(rdx).max() < 256 and np.array_equal(gdx, rdx.astype(np.float32))
        gdw = layer.dw.to_host().reshape(Ci, R, S, Co).transpose(0, 3, 1, 2)
        assert np.array_equal(gdw, rdw.astype(np.float32))
        if b is not None:
            assert np.array_equal(layer.db.to_host(), rdb.astype(np.float32))
        pre = want - (0 if b is None else b)
        ip = [float((pre * dy).sum()), float((x * gdx).sum()), float((w * gdw).sum())]
        assert ip[0] == ip[1] == ip[2]
    finally:
        layer.close()


@pytest.mark.parametrize("shape", CONVT[:5])
@pytest.mark.parametrize("act", [0, 1, 3])
def test_convt_random_operands_bounded(pkg, eng, shape, act):
    """y, dx and dw on random operands within the wide family's bounds of the float64 reference; reruns bit-identical"""
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    rng = np.random.default_rng(7 + act)
    x = rng.standard_normal((N, H, W, Ci)).astype(np.float32)
    w = (rng.standard_normal((Ci, Co, R, S)) / np.sqrt(Ci * R * S / st ** 2)).astype(np.float32)
    b = rng.standard_normal(Co).astype(np.float32)
    layer = _convt_layer(pkg, eng, shape, w, b, act)
    try:
        _, Ho, Wo, _ = layer.out_shape
        xd = dev_bits(pkg.f32_to_bf16_bits(x))
        y, again = nan_buf(N * Ho * Wo * Co), nan_buf(N * Ho * Wo * Co)
        layer.forward(xd, y)
        layer.forward(xd, again)
        eng.sync()
        assert np.array_equal(host(again), host(y))
        dy = dev_bits(pkg.f32_to_bf16_bits(rng.standard_normal((N, Ho, Wo, Co)).astype(np.float32)))
        dpre = dev_bits(dpre_of(pkg, y, dy, act, (N, Ho, Wo, Co)))
        dx, dx2 = nan_buf(N * H * W * Ci), nan_buf(N * H * W * Ci)
        layer.backward(y, dy.clone(), dx)
        dw = layer.dw.to_host()
        layer.backward(y, dy.clone(), dx2)
        eng.sync()
        assert np.array_equal(host(dx), host(dx2)) and np.array_equal(dw, layer.dw.to_host())
        check_convt(pkg, layer, xd, y, dpre, dx)
    finally:
        layer.close()


@pytest.mark.parametrize("shape", CONVT[:5])
def test_convt_without_bias_is_the_wide_input_gradient(pkg, eng, shape):
    """no bias, act 0: bit for bit pcnn_conv_wide_dgrad_padded of the adjoint convolution on the same operands"""
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    rng = np.random.default_rng(11)
    x = rng.standard_normal((N, H, W, Ci)).astype(np.float32)
    w = rng.standard_normal((Ci, Co, R, S)).astype(np.float32)
    layer = _convt_layer(pkg, eng, shape, w)
    try:
        _, Ho, Wo, _ = layer.out_shape
        xd = dev_bits(pkg.f32_to_bf16_bits(x))
        y, ref = nan_buf(N * Ho * Wo * Co), nan_buf(N * Ho * Wo * Co)
        layer.forward(xd, y)
        eng.conv_wide_dgrad(xd, layer.filt, ref, N, Ho, Wo, Co, Ci, R, S, Wo * Co, 0, st, pad)
        eng.sync()
        assert np.array_equal(host(y), host(ref))
    finally:
        layer.close()


def test_convt_after_an_optimizer_step_matches_a_fresh_layer(pkg, eng):
    shape = CONVT[0]
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    rng = np.random.default_rng(5)
    x = rng.standard_normal((N, H, W, Ci)).astype(np.float32)
    w, b = rng.standard_normal((Ci, Co, R, S)).astype(np.float32) * 0.1, rng.standard_normal(Co).astype(np.float32)
    layer = _convt_layer(pkg, eng, shape, w, b, act=3)
    opt = pkg.SGD(eng, [layer], momentum=0.9)
    fresh = None
    try:
        _, Ho, Wo, _ = layer.out_shape
        xd = dev_bits(pkg.f32_to_bf16_bits(x))
        dyd = dev_bits(pkg.f32_to_bf16_bits(rng.standard_normal((N, Ho, Wo, Co)).astype(np.float32)))
        y, dx = nan_buf(N * Ho * Wo * Co), nan_buf(N * H * W * Ci)
        for _ in range(2):
            layer.forward(xd, y)
            layer.backward(y, dyd.clone(), dx)
            opt.step(0.05)
        eng.sync()
        fresh = _convt_layer(pkg, eng, shape, layer.weight(), layer.bias.to_host(), act=3)
        y1, y2 = nan_buf(N * Ho * Wo * Co), nan_buf(N * Ho * Wo * Co)
        dx1, dx2 = nan_buf(N * H * W * Ci), nan_buf(N * H * W * Ci)
        layer.forward(xd, y1)
        fresh.forward(xd, y2)
        layer.backward(y1, dyd.clone(), dx1)
        fresh.backward(y2, dyd.clone(), dx2)
        eng.sync()
        assert np.array_equal(host(y1), host(y2)) and np.array_equal(host(dx1), host(dx2))
    finally:
        opt.close()
        layer.close()
        if fresh:
            fresh.close()


def test_convt_refusals(pkg, eng):
    w = np.zeros((16, 8, 4, 4), np.float32)
    with pytest.raises(pkg.PcnnError, match="output_padding"):
        pkg.ConvTransposeLayer(eng, 1, 4, 4, 16, 8, 4, 4, w, stride=2, output_padding=(2, 0))
    with pytest.raises(pkg.PcnnError, match="y must be dense"):
        pkg.ConvTransposeLayer(eng, 1, 4, 4, 16, 8, 4, 4, w, np.zeros(8), stride=2, padding=(1, 1), row_pitch=72)
    with pytest.raises(pkg.PcnnError, match="C_in"):
        eng.conv_transpose_fwd(1, 1, None, 1, 1, 4, 4, 12, 8, 4, 4, 2)
    with pytest.raises(pkg.PcnnError, match="NULL"):
        eng.conv_transpose_fwd(None, 1, None, 1, 1, 4, 4, 16, 8, 4, 4, 2)


RESIZE = [(2, 7, 7, 11, 28, 28), (2, 7, 7, 16, 14, 14), (1, 8, 8, 8, 64, 64), (2, 28, 28, 8, 7, 7), (1, 10, 13, 3, 6, 17),
          (1, 5, 5, 8, 5, 5), (1, 1, 3, 5, 4, 1), (4, 28, 28, 32, 56, 56)]


@pytest.mark.parametrize("N,H,W,C,Ho,Wo", RESIZE)
def test_upsample_bit_identical_to_replay(pkg, eng, N, H, W, C, Ho, Wo):
    rng = np.random.default_rng(H * Ho + C)
    x = rng.standard_normal((N, H, W, C)).astype(np.float32)
    x.reshape(-1)[:6] = [np.inf, -np.inf, np.nan, 0.0, -0.0, 1e-40][:x.size]
    xb = SR.bf16_bits(x)
    layer = pkg.UpsampleBilinearLayer(eng, N, H, W, C, Ho, Wo)
    y = guarded(N * Ho * Wo * C)
    layer.forward(dev_bits(xb), y)
    dy = rng.standard_normal((N, Ho, Wo, C)).astype(np.float32)
    dy.reshape(-1)[:5] = [np.inf, -0.0, np.nan, -np.inf, 0.0][:dy.size]
    dyb = SR.bf16_bits(dy)
    dx, dx2 = guarded(N * H * W * C), guarded(N * H * W * C)
    layer.backward(dev_bits(dyb), dx)
    layer.backward(dev_bits(dyb), dx2)
    eng.sync()
    yb, dxb = host(y), host(dx)
    assert np.all(yb[-64:] == NAN) and np.all(dxb[-64:] == NAN)
    assert np.array_equal(yb[:-64], SR.upsample_fwd_replay(xb, Ho, Wo).reshape(-1))
    assert np.array_equal(dxb[:-64], SR.upsample_bwd_replay(dyb, H, W).reshape(-1))
    assert np.array_equal(dxb, host(dx2))


def test_upsample_close_to_torch(pkg, eng):
    N, H, W, C, Ho, Wo = 4, 7, 7, 16, 28, 28
    rng = np.random.default_rng(2)
    xb = pkg.f32_to_bf16_bits(rng.standard_normal((N, H, W, C)).astype(np.float32))
    xt = torch.from_numpy(pkg.bf16_bits_to_f32(xb)).to(DEV).permute(0, 3, 1, 2).requires_grad_(True)
    yt = torch.nn.functional.interpolate(xt, size=(Ho, Wo), mode="bilinear", align_corners=False)
    dyb = pkg.f32_to_bf16_bits(rng.standard_normal((N, Ho, Wo, C)).astype(np.float32))
    yt.backward(torch.from_numpy(pkg.bf16_bits_to_f32(dyb)).to(DEV).permute(0, 3, 1, 2))
    y, dx = nan_buf(N * Ho * Wo * C), nan_buf(N * H * W * C)
    eng.upsample_bilinear_fwd(dev_bits(xb), y, N, H, W, C, Ho, Wo)
    eng.upsample_bilinear_bwd(dev_bits(dyb), dx, N, H, W, C, Ho, Wo)
    eng.sync()
    ty = yt.detach().permute(0, 2, 3, 1).cpu().numpy()
    tdx = xt.grad.permute(0, 2, 3, 1).cpu().numpy()
    assert np.all(np.abs(pkg.bf16_bits_to_f32(host(y)).reshape(ty.shape) - ty) <= 2 ** -8 * np.abs(ty) + 1e-6)
    assert np.all(np.abs(pkg.bf16_bits_to_f32(host(dx)).reshape(tdx.shape) - tdx) <= 2 ** -8 * np.abs(tdx) + 1e-5)


def test_upsample_refusals(pkg, eng):
    with pytest.raises(pkg.PcnnError, match="16-byte"):
        eng.upsample_bilinear_fwd(2, 4096, 1, 2, 2, 8, 4, 4)
    with pytest.raises(pkg.PcnnError, match="overlap"):
        eng.upsample_bilinear_fwd(4096, 4096, 1, 2, 2, 8, 4, 4)
    with pytest.raises(pkg.PcnnError, match="NULL"):
        eng.upsample_bilinear_bwd(None, 4096, 1, 2, 2, 8, 4, 4)


@pytest.mark.parametrize("case", ["mixed", "all_ignored", "no_ignore", "nonfinite", "big_target"])
def test_pixel_ce(pkg, eng, case):
    rng = np.random.default_rng(len(case))
    P, O = 5000, 11
    z = (rng.standard_normal((P, O)) * 3).astype(np.float32)
    t = rng.integers(0, O, P).astype(np.uint8)
    ii = 255
    if case != "no_ignore":
        t[rng.random(P) < 0.3] = 255
    if case == "all_ignored":
        t[:] = 255
    if case == "no_ignore":
        ii = -1
    if case == "nonfinite":
        z[3, 2], z[4, 5], z[5, 0], z[6, 1] = np.inf, -np.inf, np.nan, np.nan
        t[6] = 255
    if case == "big_target":
        t[7] = 20
    zb = pkg.f32_to_bf16_bits(z)
    d = guarded(P * O)
    loss = torch.full((P + 16,), float("nan"), device=DEV)
    pred = torch.full((P,), -7, dtype=torch.int32, device=DEV)
    count = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    td = torch.from_numpy(t).to(DEV)
    eng.softmax_ce_pixels_bf16(dev_bits(zb), td, P, O, ii, d, count, loss, pred)
    eng.sync()
    db, lh, ph, cnt = host(d), loss.cpu().numpy(), pred.cpu().numpy(), int(count.item())
    assert np.all(db[-64:] == NAN) and np.all(np.isnan(lh[P:]))
    g, rl, rp, rc, mean = SR.ce_pixels_f64(pkg.bf16_bits_to_f32(zb), t, ii)
    assert cnt == rc and np.array_equal(ph, rp)
    ign = t == ii
    assert np.all(db[:-64].reshape(P, O)[ign] == 0) and np.all(lh[:P][ign] == 0)
    # every non-ignored row is the hard call's row at the device's scale, bit for bit
    if rc:
        ref = nan_buf(P * O)
        ref_loss = torch.full((P,), float("nan"), device=DEV)
        eng.softmax_ce_bf16(dev_bits(zb), td, P, O, float(np.float32(1.0 / rc)), ref, ref_loss)
        eng.sync()
        assert np.array_equal(db[:-64].reshape(P, O)[~ign], host(ref).reshape(P, O)[~ign])
        rlh = ref_loss.cpu().numpy()
        assert np.array_equal(lh[:P][~ign].view(np.uint32), rlh[~ign].view(np.uint32))
        want = linear_ref.f64_to_bf16_bits(pkg, g)
        near = linear_ref.near_boundary(pkg, g)
        got = db[:-64].reshape(P, O)
        assert np.all((got == want) | near | (np.isnan(g) & np.isnan(pkg.bf16_bits_to_f32(got))))
    else:                                     # every row ignored: no NaN anywhere, every dlogit +0 and every loss 0
        assert cnt == 0 and np.all(db[:-64] == 0) and np.all(lh[:P].view(np.uint32) == 0)
    # in place, rerun
    zi = dev_bits(zb)
    eng.softmax_ce_pixels_bf16(zi, td, P, O, ii, zi, count)
    eng.sync()
    assert np.array_equal(host(zi).reshape(-1), db[:-64])


def test_pixel_ce_refusals(pkg, eng):
    z = nan_buf(8 * 11)
    t = torch.zeros(8, dtype=torch.uint8, device=DEV)
    c = torch.zeros(1, dtype=torch.int32, device=DEV)
    for args, msg in (((z, t, 8, 11, 256, z, c), "ignore_index"), ((z, t, 8, 257, 255, z, c), "O = 257"),
                      ((z, t, 0, 11, 255, z, c), "pixels = 0"), ((z, t, 8, 11, 255, z, None), "NULL")):
        with pytest.raises(pkg.PcnnError, match=msg):
            eng.softmax_ce_pixels_bf16(*args)
    with pytest.raises(pkg.PcnnError, match="overlaps"):
        eng.softmax_ce_pixels_bf16(z, t, 8, 11, 255, z.data_ptr() + 2, c)


def test_mask_batch(pkg, eng):
    rng = np.random.default_rng(9)
    n, H, W, N = 300, 28, 28, 64
    images = rng.integers(0, 256, (n, H, W)).astype(np.uint8)
    masks = rng.integers(0, 12, (n, H, W)).astype(np.uint8)
    plain = pkg.ImageBatcher(eng, images, None, N, pad=2, flip=True, seed=3, C_out=8)
    withm = pkg.ImageBatcher(eng, images, None, N, pad=2, flip=True, seed=3, C_out=8, masks=masks)
    try:
        for epoch, step in ((0, 0), (2, 3)):
            plain.epoch = withm.epoch = epoch
            xp, _ = plain.batch(step)
            xm, _, mo = withm.batch(step)
            eng.sync()
            assert np.array_equal(plain.x.to_host(), withm.x.to_host())
            want, i, oy, ox, fl = SR.mask_batch(masks, step * N, N, 1, 2, 1, 3, epoch)
            got = mo.to_host().reshape(N, H, W)
            assert np.array_equal(got, want)
            assert np.array_equal(got, SR.torchvision_masks(masks, i, oy, ox, fl, 2))
        _, _, mo = withm.batch(1, training=False)
        eng.sync()
        assert np.array_equal(mo.to_host().reshape(N, H, W), masks[N:2 * N])
    finally:
        plain.close()
        withm.close()
    with pytest.raises(pkg.PcnnError, match="mask_fill"):
        eng.augment_mask(1, n, H, W, 0, N, 1, shuffle=1, pad=2, mask_fill=300)
    with pytest.raises(pkg.PcnnError, match="pad = 65"):
        eng.augment_mask(1, n, H, W, 0, N, 2 ** 40, pad=65)


# test mIoU of the float32 torch CPU replicas on the same batches (scripts/fcn_replica.py); the device must come within 0.05
REPLICA_MIOU = {"FCNLite": 0.2459, "FCNBilinear": 0.1913}


@pytest.mark.parametrize("name", ["FCNLite", "FCNBilinear"])
def test_segmenter_trains(pkg, eng, golden, name):
    cls = getattr(segment_nets, name)

    def check_step(net, it, x, labels, masks):
        net.forward(x, labels, masks)
        eng.sync()
        P = net.pixels
        t = masks.to_host().reshape(-1)
        keep = t != segment_nets.IGNORE
        cnt = int(net.count.item())
        assert cnt == int(keep.sum())
        # the pixel loss: non-ignored rows are the hard call's at scale RN32(1 / count), bit for bit; ignored rows +0 and 0
        ref, ref_loss = nan_buf(P * 11), torch.full((P,), float("nan"), device=DEV)
        eng.softmax_ce_bf16(net.z, masks, P, 11, float(np.float32(1.0 / cnt)), ref, ref_loss)
        eng.sync()
        dz, lh = host(net.dz).reshape(P, 11), net.loss.cpu().numpy()
        assert np.array_equal(dz[keep], host(ref).reshape(P, 11)[keep]) and np.all(dz[~keep] == 0)
        assert np.array_equal(lh[keep].view(np.uint32), ref_loss.cpu().numpy()[keep].view(np.uint32)) and np.all(lh[~keep] == 0)
        if name == "FCNLite":
            check_convt(pkg, net.t1, net.c, net.y4)
            check_convt(pkg, net.t2, net.d, net.y5)
        else:
            assert np.array_equal(host(net.z).reshape(-1), SR.upsample_fwd_replay(host(net.z7).reshape(net.NB, 7, 7, 11), 28, 28).reshape(-1))
        net.backward()
        eng.sync()
        if name == "FCNLite":
            # no bias and act 0: the gradient each transposed convolution consumed is its dy buffer, unchanged by its backward
            check_convt(pkg, net.t1, net.c, net.y4, net.dy4, net.dc)
            check_convt(pkg, net.t2, net.d, net.y5, net.dy5, net.dd)
        else:
            assert np.array_equal(host(net.dz7).reshape(-1), SR.upsample_bwd_replay(host(net.dz).reshape(net.NB, 28, 28, 11), 7, 7).reshape(-1))

    losses, miou, bg, _ = segment_nets.train_segmenter(eng, pkg, golden, cls, check_step)
    print(f"{name}: epoch losses {losses}, test mIoU {miou:.4f}, all-background mIoU {bg:.4f}")
    assert losses[-1] < losses[0]
    assert abs(miou - REPLICA_MIOU[name]) <= 0.05 and miou > 2 * bg
    _, again, _, _ = segment_nets.train_segmenter(eng, pkg, golden, cls)
    assert again == miou
