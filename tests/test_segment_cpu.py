"""Host-only checks of the dense-prediction references (segment_ref.py) against torch's CPU float64 operators and autograd, of the
float32 replays against those references, of the mask replay against torchvision, and of the host queries' domains."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import segment_ref as SR


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).double().requires_grad_(True)


CONVT = [  # N, H, W, C_in, C_out, R, S, stride, padding, output_padding
    (2, 3, 4, 8, 8, 3, 3, 1, (0, 0), (0, 0)),
    (2, 4, 3, 16, 8, 4, 4, 2, (1, 1), (0, 0)),
    (1, 5, 5, 8, 16, 3, 3, 2, (1, 1), (1, 1)),
    (1, 3, 4, 8, 8, 2, 3, 3, (0, 1), (2, 1)),
    (2, 2, 3, 8, 8, 3, 2, 4, (2, 1), (3, 0)),      # stride > taps: pixels no window reaches
    (1, 4, 4, 8, 8, 1, 1, 2, (0, 0), (1, 1)),
]


@pytest.mark.parametrize("shape", CONVT)
@pytest.mark.parametrize("act", [0, 1, 3])
def test_convt_reference_matches_torch(shape, act):
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    rng = np.random.default_rng(sum(shape[:8]) + act)
    x, w, b = rng.standard_normal((N, H, W, Ci)), rng.standard_normal((Ci, Co, R, S)), rng.standard_normal(Co)
    xt, wt, bt = _t(x.transpose(0, 3, 1, 2)), _t(w), _t(b)
    pre_t = F.conv_transpose2d(xt, wt, bt, stride=st, padding=pad, output_padding=op)
    y_t = {0: pre_t, 1: torch.sigmoid(pre_t), 3: torch.relu(pre_t)}[act]
    dy = rng.standard_normal(tuple(y_t.shape))
    y_t.backward(torch.from_numpy(dy))
    pre, y = SR.convt_fwd_f64(x, w, b, st, pad, op, act)
    assert y.shape[1:3] == SR.convt_out(H, W, R, S, st, pad, op)
    np.testing.assert_allclose(y, y_t.detach().numpy().transpose(0, 2, 3, 1), rtol=0, atol=1e-12)
    dyn = dy.transpose(0, 2, 3, 1)
    dpre = {0: dyn, 1: dyn * y * (1 - y), 3: np.where(pre > 0, dyn, 0.0)}[act]
    dx, dw, db = SR.convt_bwd_f64(x, w, dpre, st, pad)
    np.testing.assert_allclose(dx, xt.grad.numpy().transpose(0, 2, 3, 1), rtol=0, atol=1e-12)
    np.testing.assert_allclose(dw, wt.grad.numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(db, bt.grad.numpy(), rtol=0, atol=1e-12)


RESIZE = [(7, 7, 28, 28), (4, 5, 8, 10), (3, 3, 24, 24), (28, 28, 7, 7), (10, 13, 6, 4), (5, 5, 5, 5), (1, 3, 4, 1), (6, 7, 13, 3)]


@pytest.mark.parametrize("H,W,Ho,Wo", RESIZE)
def test_upsample_reference_matches_torch(H, W, Ho, Wo):
    rng = np.random.default_rng(H * 100 + Wo)
    x = rng.standard_normal((2, H, W, 3))
    xt = _t(x.transpose(0, 3, 1, 2))
    yt = F.interpolate(xt, size=(Ho, Wo), mode="bilinear", align_corners=False)
    dy = rng.standard_normal(tuple(yt.shape))
    yt.backward(torch.from_numpy(dy))
    np.testing.assert_allclose(SR.upsample_fwd_f64(x, Ho, Wo), yt.detach().numpy().transpose(0, 2, 3, 1), rtol=0, atol=1e-12)
    np.testing.assert_allclose(SR.upsample_bwd_f64(dy.transpose(0, 2, 3, 1), H, W), xt.grad.numpy().transpose(0, 2, 3, 1), rtol=0, atol=1e-12)


@pytest.mark.parametrize("H,W,Ho,Wo", RESIZE)
def test_upsample_replays_within_float32(H, W, Ho, Wo):
    """the float32 replays of both passes, on bf16 operands, are within bf16 rounding of the float64 references"""
    rng = np.random.default_rng(H + W)
    xb = SR.bf16_bits(rng.standard_normal((2, H, W, 8)).astype(np.float32))
    y = SR.bits_f32(SR.upsample_fwd_replay(xb, Ho, Wo)).astype(np.float64)
    ref = SR.upsample_fwd_f64(SR.bits_f32(xb), Ho, Wo)
    assert np.all(np.abs(y - ref) <= 2.0 ** -8 * np.abs(ref) + 1e-30 + 2 ** -20 * np.abs(ref).max())
    dyb = SR.bf16_bits(rng.standard_normal((2, Ho, Wo, 8)).astype(np.float32))
    dx = SR.bits_f32(SR.upsample_bwd_replay(dyb, H, W)).astype(np.float64)
    ref = SR.upsample_bwd_f64(SR.bits_f32(dyb), H, W)
    assert np.all(np.abs(dx - ref) <= 2.0 ** -8 * np.abs(ref) + 2 ** -16 * np.abs(ref).max())


@pytest.mark.parametrize("H,W,Ho,Wo", [(3, 3, 3, 6), (3, 4, 7, 4), (4, 4, 4, 4), (5, 3, 2, 3)])
def test_upsample_replay_nonfinite_as_torch_cpu(H, W, Ho, Wo):
    """with an axis unchanged, torch's CPU kernel copies along it (per axis), as the device does: on +-Inf and NaN inputs the
    replay's NaN pattern and values equal torch's float32 CPU result within rounding"""
    rng = np.random.default_rng(H * Wo)
    x = rng.standard_normal((1, H, W, 8)).astype(np.float32)
    x[0, 1, 1, 0], x[0, 0, W - 1, 1], x[0, H - 1, 0, 2] = np.inf, -np.inf, np.nan
    xb = SR.bf16_bits(x)
    y = SR.bits_f32(SR.upsample_fwd_replay(xb, Ho, Wo)).astype(np.float64)
    t = F.interpolate(torch.from_numpy(SR.bits_f32(xb)).permute(0, 3, 1, 2), size=(Ho, Wo), mode="bilinear", align_corners=False)
    t = t.permute(0, 2, 3, 1).numpy().astype(np.float64)
    assert np.array_equal(np.isnan(y), np.isnan(t))
    fin = np.isfinite(t)
    assert np.array_equal(np.isinf(y), np.isinf(t)) and np.array_equal(y[np.isinf(t)], t[np.isinf(t)])
    assert np.all(np.abs(y[fin] - t[fin]) <= 2 ** -8 * np.abs(t[fin]) + 1e-6)


@pytest.mark.parametrize("case", ["mixed", "none_ignored", "all_ignored", "nonfinite", "no_ignore_index"])
def test_pixel_ce_reference_matches_torch(case):
    rng = np.random.default_rng(len(case))
    P, O = 300, 11
    z = rng.standard_normal((P, O)) * 3
    t = rng.integers(0, O, P).astype(np.uint8)
    ii = 255
    if case == "mixed":
        t[rng.random(P) < 0.3] = 255
    elif case == "all_ignored":
        t[:] = 255
    elif case == "no_ignore_index":
        ii = -1
    elif case == "nonfinite":
        t[rng.random(P) < 0.3] = 255
        z[3, 2], z[4, 5], z[5, 0] = np.inf, -np.inf, np.nan
    g, loss, pred, count, mean = SR.ce_pixels_f64(z, t, ii)
    zt = _t(z)
    lt = F.cross_entropy(zt, torch.from_numpy(t.astype(np.int64)), ignore_index=ii if ii >= 0 else -100)
    assert count == int((t != ii).sum())
    if count == 0:
        assert np.isnan(mean) and np.isnan(float(lt.detach())) and np.all(g == 0) and not np.signbit(g).any()
        return
    lt.backward()
    finite = np.isfinite(z).all(axis=1)
    if finite.all():
        np.testing.assert_allclose(mean, float(lt.detach()), rtol=1e-12)
    ok = finite | (t == ii)
    # torch's mean divides by the float count; the reference scales by fp32(1 / count): equal within fp32's rounding of 1 / count
    np.testing.assert_allclose(g[ok], zt.grad.numpy()[ok], rtol=2 ** -23, atol=1e-15)
    assert np.all(g[t == ii] == 0) and np.all(loss[t == ii] == 0)


def test_mask_replay_matches_torchvision():
    rng = np.random.default_rng(3)
    masks = rng.integers(0, 12, (40, 9, 11)).astype(np.uint8)
    for pad, flip, epoch in ((2, 1, 0), (4, 0, 3), (0, 1, 1), (3, 1, 7)):
        got, i, oy, ox, fl = SR.mask_batch(masks, 8, 16, 1, pad, flip, seed=11, epoch=epoch)
        assert np.array_equal(got, SR.torchvision_masks(masks, i, oy, ox, fl, pad))
    got, i, _, _, _ = SR.mask_batch(masks, 4, 10, 0, 0, 0)
    assert np.array_equal(got, masks[4:14])


def test_digit_masks():
    u8 = np.array([[0, 31, 32, 127, 128, 255] + [0] * 778], np.uint8)
    m = SR.digit_masks(u8, np.array([7]))
    assert list(m.reshape(-1)[:6]) == [0, 0, 255, 255, 8, 8]


def test_convt_info_domain(pkg):
    i = pkg.conv_transpose_info(128, 7, 7, 64, 32, 4, 4, 2, (1, 1))
    assert (i["H_out"], i["W_out"], i["row_pitch"], i["image_rows"]) == (14, 14, 14 * 32, 14)
    i = pkg.conv_transpose_info(2, 5, 5, 8, 16, 3, 3, 2, (1, 1), (1, 1), bias=True, act=3)
    assert (i["H_out"], i["W_out"]) == (10, 10)


@pytest.mark.parametrize("change,msg", [
    (dict(C_in=12), "C_in"), (dict(C_in=264), "C_in"), (dict(C_out=12), "C_out"), (dict(C_out=264, bias=True), "C_out = 264 with a bias"),
    (dict(act=2), "act 2"), (dict(stride=5), "stride 5"), (dict(R=8), "taps"), (dict(padding=(4, 1)), "padding"),
    (dict(output_padding=(2, 0)), "output_padding"), (dict(row_pitch=12), "row pitch"), (dict(N=0), "N = 0"),
])
def test_convt_info_refusals(pkg, change, msg):
    a = dict(N=2, H=5, W=5, C_in=16, C_out=32, R=4, S=4, stride=2, padding=(1, 1), output_padding=(0, 0), row_pitch=None, image_rows=0,
             bias=False, act=0)
    a.update(change)
    with pytest.raises(pkg.PcnnError, match=msg):
        pkg.conv_transpose_info(**a)


def test_convt_info_wide_c_out_without_bias(pkg):
    assert pkg.conv_transpose_info(1, 4, 4, 16, 264, 4, 4, 2, (1, 1))["groups"] == 2


def test_upsample_info(pkg):
    assert pkg.upsample_bilinear_info(2, 7, 7, 16, 28, 28)["vec"] == 8
    assert pkg.upsample_bilinear_info(2, 7, 7, 3, 28, 28)["vec"] == 1
    for args, msg in (((0, 7, 7, 8, 28, 28), "N = 0"), ((1, 0, 7, 8, 28, 28), "H = 0"), ((1, 7, 7, 8, 0, 28), "H_out = 0"),
                      ((1, 7, 7, 8, 16385, 28), "16384"), ((1, 7, 7, 0, 28, 28), "C = 0")):
        with pytest.raises(pkg.PcnnError, match=msg):
            pkg.upsample_bilinear_info(*args)


def test_batcher_refuses_masks_outside_the_plain_path(pkg):
    images = np.zeros((8, 6, 6), np.uint8)
    masks = np.zeros((8, 6, 6), np.uint8)
    for kw, msg in ((dict(crop_size=4), "masks with crop_size"), (dict(random_erase=0.5), "masks with"), (dict(mixup_alpha=0.2), "masks with")):
        with pytest.raises(pkg.PcnnError, match=msg):
            pkg.ImageBatcher(None, images, None, 4, masks=masks, **kw)
    with pytest.raises(pkg.PcnnError, match="masks must be uint8"):
        pkg.ImageBatcher(None, images, None, 4, masks=np.zeros((8, 6, 5), np.uint8))
    with pytest.raises(pkg.PcnnError, match="mask_fill"):
        pkg.ImageBatcher(None, images, None, 4, masks=masks, mask_fill=256)


def test_segmentation_scores():
    t = np.array([0, 0, 1, 1, 2, 255, 2])
    p = np.array([0, 1, 1, 1, 0, 2, -1])
    import pcnn_loader
    conf, iou, miou = pcnn_loader.load().segmentation_scores(p, t, 3, 255)
    assert conf.tolist() == [[1, 1, 0], [0, 2, 0], [1, 0, 0]]
    np.testing.assert_allclose(iou, [1 / 3, 2 / 3, 0.0])
    assert miou == pytest.approx(1 / 3)
