"""Dense prediction at the sizes scripts/conv_bench.py times it (convt, upsample, segce), where the kernels loop: the transposed
convolution over many tiles per CTA, over split weight-gradient slots, with two channel groups and into pitched outputs; the
per-pixel cross-entropy past the first grid-stride lap of both of its kernels; and the bilinear resize at the benchmark's shapes and
past its 2^20-block grid cap.  Every shape asserts the coverage it exists for from the host-only info queries, so that a plan change
cannot shrink it unnoticed.  The float64 references of the transposed convolution are torch's CPU operators (equal to segment_ref's,
test_segment_scale_cpu.py); the pixel loss is compared with segment_ref.ce_pixels_f64 and the resize with its float32 replays."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import linear_ref
import segment_ref as SR
from example_nets import DEV, host, nan_buf
from test_segment_gpu import NAN, dev_bits, dpre_of, guarded, ints

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ transposed convolution
CONVT_SCALE = [  # N, H, W, C_in, C_out, R, S, stride, padding, output_padding
    (128, 7, 7, 256, 128, 4, 4, 2, (1, 1), (0, 0)),     # the three decoder shapes of conv_bench.py convt
    (128, 14, 14, 128, 64, 4, 4, 2, (1, 1), (0, 0)),
    (128, 28, 28, 64, 32, 4, 4, 2, (1, 1), (0, 0)),
    (128, 7, 7, 64, 24, 3, 3, 2, (1, 1), (1, 1)),       # C_out 24: padded MMA columns on every tile
    (64, 8, 8, 32, 16, 2, 2, 3, (1, 0), (2, 1)),        # taps < stride: some phases have no tap, on later tiles too
    (64, 6, 6, 256, 264, 3, 3, 1, (1, 1), (0, 0)),      # two channel groups
]
CONVT_IDS = [f"{s[0]}x{s[1]}x{s[2]}x{s[3]}-{s[4]}_{s[5]}x{s[6]}s{s[7]}" for s in CONVT_SCALE]


def coverage(pkg, shape, row_pitch=None, image_rows=0):
    """tiles and channel groups of the forward (the input-gradient kernel with the epilogue); the weight gradient's splits (pixel
    ranges, one slot each) and the most pixel blocks one of its work units adds (the adjoint convolution's forward blocks per range)"""
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    i = pkg.conv_transpose_info(N, H, W, Ci, Co, R, S, st, pad, op, row_pitch, image_rows)
    adj = (N, i["H_out"], i["W_out"], Co, Ci, R, S, st, i["row_pitch"], i["image_rows"], pad)
    b = pkg.conv_wide_bwd_info(*adj)
    blocks = pkg.conv_wide_plan_info(*adj)["tiles"]
    return dict(tiles=i["tiles"], groups=i["groups"], wgrad_splits=b["wgrad_splits"], wgrad_max_blocks=-(-blocks // b["wgrad_splits"]))


def assert_coverage(pkg, shape, sm_count):
    """the weight gradient reduces more than one slot; one group runs at least three tiles on every CTA, or two groups exist"""
    c = coverage(pkg, shape)
    assert c["wgrad_splits"] > 1, (shape, c)
    if shape[4] > 256:
        assert c["groups"] == 2, (shape, c)
    else:
        assert c["groups"] == 1 and c["tiles"] >= 3 * sm_count, (shape, c)


@pytest.fixture(scope="module")
def sm_count(eng):
    return eng.device_info()["sm_count"]


def torch_convt(shape, x, w, b=None, dpre=None):
    """float64 conv_transpose2d on the CPU, NHWC in and out, w [C_in][C_out][R][S]: [pre], or with the gradient dpre at the
    pre-activation [pre, dx, dw] (dw in w's layout)"""
    _, _, _, _, _, _, _, st, pad, op = shape
    xt = torch.from_numpy(np.ascontiguousarray(np.asarray(x, np.float64).transpose(0, 3, 1, 2))).requires_grad_(dpre is not None)
    wt = torch.from_numpy(np.asarray(w, np.float64)).requires_grad_(dpre is not None)
    bt = None if b is None else torch.from_numpy(np.asarray(b, np.float64))
    pre = F.conv_transpose2d(xt, wt, bt, stride=st, padding=pad, output_padding=op)
    out = [pre.detach().permute(0, 2, 3, 1).numpy()]
    if dpre is not None:
        g = torch.from_numpy(np.ascontiguousarray(np.asarray(dpre, np.float64).transpose(0, 3, 1, 2)))
        dx, dw = torch.autograd.grad(pre, (xt, wt), g)
        out += [dx.permute(0, 2, 3, 1).numpy(), dw.numpy()]
    return out


def _layer(pkg, eng, shape, w, b=None, act=0, row_pitch=None, image_rows=0):
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    return pkg.ConvTransposeLayer(eng, N, H, W, Ci, Co, R, S, w, b, act=act, stride=st, padding=pad, output_padding=op,
                                  row_pitch=row_pitch, image_rows=image_rows)


def _f32(pkg, bits, shape):
    return pkg.bf16_bits_to_f32(bits).reshape(shape)


def _dw(layer):
    """the layer's fp32 dw in torch's layout [C_in][C_out][R][S]"""
    N, H, W, Ci, Co, R, S = layer.shape
    return layer.dw.to_host().reshape(Ci, R, S, Co).transpose(0, 3, 1, 2)


@pytest.mark.parametrize("shape", CONVT_SCALE, ids=CONVT_IDS)
def test_convt_scale_integer_operands_exact(pkg, eng, sm_count, shape):
    """y, dx, dw and db equal the float64 reference bit for bit on small sparse integers, and <pre, dy> = <x, dx> = <w, dw>
    exactly: every partial sum is an integer below 2^24 and every result below 256, so any fp32 order is exact"""
    assert_coverage(pkg, shape, sm_count)
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    rng = np.random.default_rng(sum(shape[:8]))
    dens = 0.1 if max(Ci, Co) > 64 else 0.5
    x, w = ints(rng, (N, H, W, Ci), density=dens), ints(rng, (Ci, Co, R, S), -2, 3, dens)
    b = None if Co > 256 else ints(rng, Co)
    layer = _layer(pkg, eng, shape, w, b)
    try:
        _, Ho, Wo, _ = layer.out_shape
        y = guarded(N * Ho * Wo * Co)
        layer.forward(dev_bits(pkg.f32_to_bf16_bits(x)), y)
        dy = ints(rng, (N, Ho, Wo, Co), -2, 3, dens)
        dx = guarded(N * H * W * Ci)
        layer.backward(y, dev_bits(pkg.f32_to_bf16_bits(dy)), dx)
        eng.sync()
        yb, dxb = host(y), host(dx)
        assert np.all(yb[-64:] == NAN) and np.all(dxb[-64:] == NAN)
        pre, rdx, rdw = torch_convt(shape, x, w, None, dy)
        want = pre if b is None else pre + b
        assert np.abs(want).max() < 256 and np.abs(rdx).max() < 256
        assert torch_convt(shape, np.abs(x), np.abs(w), None, np.abs(dy))[2].max() < 2 ** 24
        assert np.array_equal(_f32(pkg, yb[:-64], want.shape), want.astype(np.float32)), "y"
        gdx = _f32(pkg, dxb[:-64], rdx.shape)
        assert np.array_equal(gdx, rdx.astype(np.float32)), "dx"
        gdw = _dw(layer)
        assert np.array_equal(gdw, rdw.astype(np.float32)), "dw"
        if b is not None:
            assert np.array_equal(layer.db.to_host(), dy.sum(axis=(0, 1, 2)).astype(np.float32)), "db"
        ip = [float((pre * dy).sum()), float((x * gdx.astype(np.float64)).sum()), float((w * gdw.astype(np.float64)).sum())]
        assert ip[0] == ip[1] == ip[2], ip
    finally:
        layer.close()


CONVT_ACTS = [(s, a) for s in CONVT_SCALE for a in ((0, 1, 3) if s[4] <= 256 else (0,))]   # an activation needs C_out <= 256
CONVT_ACT_IDS = [f"{CONVT_IDS[CONVT_SCALE.index(s)]}-act{a}" for s, a in CONVT_ACTS]


@pytest.mark.parametrize("shape,act", CONVT_ACTS, ids=CONVT_ACT_IDS)
def test_convt_scale_random_operands_bounded(pkg, eng, sm_count, shape, act):
    """random operands with a bias (none for C_out > 256, which refuses it), against the float64 reference on the layer's own bf16
    operands; forward and backward reruns bit-identical, dw and db included (the split slots are reduced in a fixed order).
      y, dx: within bf16 rounding plus an fp32 accumulation term, 2^-8 |ref| + 2^-18 sum|products|.
      dw: each element is a sum over the N H W pixels of x, added 16 pixels per wgmma into one fp32 accumulator per work unit (8
          updates per pixel block, at most wgrad_max_blocks blocks), then one slot per split added in a fixed order.  Each update
          rounds by at most 2^-23 of a running value below sum|x dy|, and the tensor core's reduction of a step may round once more:
          |dw - ref| <= 2 n_acc 2^-23 sum|x dy|, n_acc = 8 wgrad_max_blocks + wgrad_splits (test_conv_wide_bwd_gpu.py's model).
          (A bound of N H W 2^-24 sum|x dy| is too loose here: dw without one of its 28 slots stays inside it.)
      db: within the fp32 bound of its sum over the N H_out W_out pixels."""
    assert_coverage(pkg, shape, sm_count)
    cov = coverage(pkg, shape)
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    rng = np.random.default_rng(7 + act + sum(shape[:8]))
    x = rng.standard_normal((N, H, W, Ci)).astype(np.float32)
    w = (rng.standard_normal((Ci, Co, R, S)) / np.sqrt(Ci * R * S / st ** 2)).astype(np.float32)
    b = None if Co > 256 else rng.standard_normal(Co).astype(np.float32)
    layer = _layer(pkg, eng, shape, w, b, act)
    try:
        _, Ho, Wo, _ = layer.out_shape
        xd = dev_bits(pkg.f32_to_bf16_bits(x))
        y, again = nan_buf(N * Ho * Wo * Co), nan_buf(N * Ho * Wo * Co)
        layer.forward(xd, y)
        layer.forward(xd, again)
        eng.sync()
        assert np.array_equal(host(again), host(y))
        dy = dev_bits(pkg.f32_to_bf16_bits(rng.standard_normal((N, Ho, Wo, Co)).astype(np.float32)))
        dpre = dpre_of(pkg, y, dy, act, (N, Ho, Wo, Co))
        dx, dx2 = nan_buf(N * H * W * Ci), nan_buf(N * H * W * Ci)
        layer.backward(y, dy.clone(), dx)
        dw = _dw(layer).copy()
        db = None if b is None else layer.db.to_host().copy()
        layer.backward(y, dy.clone(), dx2)
        eng.sync()
        assert np.array_equal(host(dx), host(dx2)) and np.array_equal(dw, _dw(layer))
        assert b is None or np.array_equal(db, layer.db.to_host())

        xq = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(x)).astype(np.float64)
        wq = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(layer.weight())).astype(np.float64)
        bq = None if b is None else b.astype(np.float64)
        dq = _f32(pkg, dpre, (N, Ho, Wo, Co)).astype(np.float64)
        pre, rdx, rdw = torch_convt(shape, xq, wq, bq, dq)
        want = SR.act_f64(pre, act)
        absum, adx, adw = torch_convt(shape, np.abs(xq), np.abs(wq), None if bq is None else np.abs(bq), np.abs(dq))
        got = _f32(pkg, host(y), want.shape).astype(np.float64)
        assert np.all(np.abs(got - want) <= 2 ** -8 * np.abs(want) + 2 ** -18 * absum + 1e-30), "y"
        gdx = _f32(pkg, host(dx), rdx.shape).astype(np.float64)
        assert np.all(np.abs(gdx - rdx) <= 2 ** -8 * np.abs(rdx) + 2 ** -18 * adx + 1e-30), "dx"
        n_acc = 8 * cov["wgrad_max_blocks"] + cov["wgrad_splits"]
        ratio = float((np.abs(dw - rdw) / (2 * n_acc * 2.0 ** -23 * adw)).max())
        print(f"convT dw {shape} act {act}: n_acc {n_acc}, worst |dw - ref| / bound = {ratio:.3e}")
        assert ratio <= 1.0, "dw"
        if b is not None:
            rdb, adb = dq.sum(axis=(0, 1, 2)), np.abs(dq).sum(axis=(0, 1, 2))
            assert np.all(np.abs(db - rdb) <= (N * Ho * Wo * 2.0 ** -24 + 2.0 ** -20) * adb + 1e-30), "db"
    finally:
        layer.close()


@pytest.mark.parametrize("shape", CONVT_SCALE, ids=CONVT_IDS)
def test_convt_scale_without_bias_is_the_wide_input_gradient(pkg, eng, sm_count, shape):
    """no bias, act 0: y bit for bit the input gradient of the adjoint convolution (the epilogue variant's accumulators and tiles are
    the plain variant's on every tile a CTA runs)"""
    assert_coverage(pkg, shape, sm_count)
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    rng = np.random.default_rng(11)
    x = rng.standard_normal((N, H, W, Ci)).astype(np.float32)
    w = rng.standard_normal((Ci, Co, R, S)).astype(np.float32)
    layer = _layer(pkg, eng, shape, w)
    try:
        _, Ho, Wo, _ = layer.out_shape
        xd = dev_bits(pkg.f32_to_bf16_bits(x))
        y, ref = guarded(N * Ho * Wo * Co), guarded(N * Ho * Wo * Co)
        layer.forward(xd, y)
        eng.conv_wide_dgrad(xd, layer.filt, ref, N, Ho, Wo, Co, Ci, R, S, Wo * Co, 0, st, pad)
        eng.sync()
        yb = host(y)
        assert np.all(yb[-64:] == NAN) and np.array_equal(yb, host(ref))
    finally:
        layer.close()


# ------------------------------------------------------------------------------------------------ pitched output
PITCHED = [  # shape, row_pitch, image_rows
    ((128, 14, 14, 128, 64, 4, 4, 2, (1, 1), (0, 0)), 1800, 30),
    ((4, 5, 6, 16, 24, 3, 3, 2, (1, 1), (1, 1)), 328, 12),
]


@pytest.mark.parametrize("shape,pitch,rows", PITCHED, ids=["128x14x14x128-64", "4x5x6x16-24"])
def test_convt_pitched_output(pkg, eng, shape, pitch, rows):
    """no bias, act 0, y at row_pitch > W_out C_out and image_rows > H_out: y is written inside each row's W_out C_out elements only
    (the NaN gaps and the rows below each image stay NaN) with the dense layer's bits; dx and dw from a dy in the same layout, NaN
    in its gaps, are the dense layer's bit for bit"""
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    rng = np.random.default_rng(pitch)
    x = rng.standard_normal((N, H, W, Ci)).astype(np.float32)
    w = (rng.standard_normal((Ci, Co, R, S)) / np.sqrt(Ci * R * S / st ** 2)).astype(np.float32)
    pitched, dense = _layer(pkg, eng, shape, w, row_pitch=pitch, image_rows=rows), _layer(pkg, eng, shape, w)
    try:
        _, Ho, Wo, _ = dense.out_shape
        assert (pitched.row_pitch, pitched.image_rows) == (pitch, rows) and pitch > Wo * Co and pitch % 8 == 0 and rows > Ho
        assert coverage(pkg, shape, pitch, rows) == coverage(pkg, shape)
        xd = dev_bits(pkg.f32_to_bf16_bits(x))
        yp, yd = guarded(N * rows * pitch), guarded(N * Ho * Wo * Co)
        pitched.forward(xd, yp)
        dense.forward(xd, yd)
        dyb = pkg.f32_to_bf16_bits(rng.standard_normal((N, Ho, Wo * Co)).astype(np.float32))
        dyp = np.full((N, rows, pitch), NAN, np.uint16)
        dyp[:, :Ho, :Wo * Co] = dyb
        dxp, dxd = guarded(N * H * W * Ci), guarded(N * H * W * Ci)
        pitched.backward(yp, dev_bits(dyp), dxp)
        dense.backward(yd, dev_bits(dyb), dxd)
        eng.sync()
        ypb, ydb = host(yp), host(yd)
        assert np.all(ypb[-64:] == NAN) and np.all(ydb[-64:] == NAN)
        ypb = ypb[:-64].reshape(N, rows, pitch)
        assert np.array_equal(ypb[:, :Ho, :Wo * Co], ydb[:-64].reshape(N, Ho, Wo * Co))
        assert np.all(ypb[:, :Ho, Wo * Co:] == NAN) and np.all(ypb[:, Ho:] == NAN)
        assert np.array_equal(host(dxp), host(dxd)) and np.all(host(dxp)[-64:] == NAN)
        assert np.array_equal(_dw(pitched), _dw(dense))
    finally:
        pitched.close()
        dense.close()


# ------------------------------------------------------------------------------------------------ per-pixel cross-entropy
# k_count_targets runs at most 4 CTAs of 256 threads per SM, one pixel per thread and lap; k_softmax_ce_bf16<false, true> at most
# 8 CTAs of 8 warps per SM, one row per warp and lap
def count_laps(P, sm_count):
    return -(-P // (min(-(-P // 256), 4 * sm_count) * 256))


def ce_laps(P, sm_count):
    return -(-P // (min(-(-P * 32 // 256), 8 * sm_count) * 8))


PIXEL_CE = [  # case, pixels, classes
    ("mixed", 16 * 224 * 224, 21),       # conv_bench.py segce
    ("mixed", 150_000, 1),
    ("mixed", 150_000, 33),
    ("mixed", 150_000, 256),
    ("no_ignore_index", 150_000, 33),
    ("last_pixel_only", 150_000, 33),
    ("all_ignored", 150_000, 33),
]


@pytest.mark.parametrize("case,P,O", PIXEL_CE, ids=[f"{c}-{p}x{o}" for c, p, o in PIXEL_CE])
def test_pixel_ce_past_the_first_lap(pkg, eng, sm_count, case, P, O):
    """the count exactly, pred exactly, dlogits within the documented rounding of segment_ref.ce_pixels_f64, non-ignored rows the
    hard call's bits at RN32(1 / count) and ignored rows +0 and 0, with ignored rows on every lap of both kernels"""
    assert P > 4 * sm_count * 256 and count_laps(P, sm_count) >= 2 and ce_laps(P, sm_count) >= 2
    rng = np.random.default_rng(P + O + len(case))
    z = (rng.standard_normal((P, O)) * 3).astype(np.float32)
    t = rng.integers(0, O, P).astype(np.uint8)
    ii = 255
    if case == "mixed":
        t[rng.random(P) < 0.1] = 255
    elif case == "no_ignore_index":
        ii = -1
    elif case == "last_pixel_only":
        t[:-1] = 255
    elif case == "all_ignored":
        t[:] = 255
    zb = pkg.f32_to_bf16_bits(z)
    td = torch.from_numpy(t).to(DEV)
    d = guarded(P * O)
    loss = torch.full((P + 16,), float("nan"), device=DEV)
    pred = torch.full((P,), -7, dtype=torch.int32, device=DEV)
    count = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    eng.softmax_ce_pixels_bf16(dev_bits(zb), td, P, O, ii, d, count, loss, pred)
    eng.sync()
    db, lh, ph, cnt = host(d), loss.cpu().numpy(), pred.cpu().numpy(), int(count.item())
    assert np.all(db[-64:] == NAN) and np.all(np.isnan(lh[P:]))
    db, lh = db[:-64].reshape(P, O), lh[:P]
    g, _, rp, rc, _ = SR.ce_pixels_f64(pkg.bf16_bits_to_f32(zb), t, ii)
    assert cnt == rc == {"no_ignore_index": P, "last_pixel_only": 1, "all_ignored": 0}.get(case, rc)
    assert np.array_equal(ph, rp)
    ign = t == ii
    assert np.all(db[ign] == 0) and np.all(lh[ign].view(np.uint32) == 0)
    if rc:
        ref = nan_buf(P * O)
        ref_loss = torch.full((P,), float("nan"), device=DEV)
        eng.softmax_ce_bf16(dev_bits(zb), td, P, O, float(np.float32(1.0 / rc)), ref, ref_loss)
        eng.sync()
        assert np.array_equal(db[~ign], host(ref).reshape(P, O)[~ign])
        assert np.array_equal(lh[~ign].view(np.uint32), ref_loss.cpu().numpy()[~ign].view(np.uint32))
        assert np.all((db == linear_ref.f64_to_bf16_bits(pkg, g)) | linear_ref.near_boundary(pkg, g))
    else:                                     # every row ignored: no NaN anywhere, every dlogit +0 and every loss 0
        assert np.all(db == 0) and np.all(lh.view(np.uint32) == 0)


# ------------------------------------------------------------------------------------------------ bilinear resize
UPSAMPLE_BENCH = [(128, 28, 28, 64, 2), (64, 28, 28, 21, 4), (32, 28, 28, 21, 8)]   # conv_bench.py upsample: N, H, W, C, factor


@pytest.mark.parametrize("N,H,W,C,f", UPSAMPLE_BENCH, ids=[f"{n}x{h}x{w}x{c}-x{f}" for n, h, w, c, f in UPSAMPLE_BENCH])
def test_upsample_benchmark_shapes_bit_identical_to_replay(pkg, eng, N, H, W, C, f):
    """forward and backward bit for bit segment_ref's replays, guard elements untouched, reruns bit-identical"""
    Ho, Wo = H * f, W * f
    rng = np.random.default_rng(N + C + f)
    xb = SR.bf16_bits(rng.standard_normal((N, H, W, C), dtype=np.float32))
    dyb = SR.bf16_bits(rng.standard_normal((N, Ho, Wo, C), dtype=np.float32))
    layer = pkg.UpsampleBilinearLayer(eng, N, H, W, C, Ho, Wo)
    y, y2 = guarded(N * Ho * Wo * C), guarded(N * Ho * Wo * C)
    dx, dx2 = guarded(N * H * W * C), guarded(N * H * W * C)
    layer.forward(dev_bits(xb), y)
    layer.forward(dev_bits(xb), y2)
    layer.backward(dev_bits(dyb), dx)
    layer.backward(dev_bits(dyb), dx2)
    eng.sync()
    yb, dxb = host(y), host(dx)
    assert np.all(yb[-64:] == NAN) and np.all(dxb[-64:] == NAN)
    assert np.array_equal(yb, host(y2)) and np.array_equal(dxb, host(dx2))
    assert np.array_equal(yb[:-64], SR.upsample_fwd_replay(xb, Ho, Wo).reshape(-1))
    assert np.array_equal(dxb[:-64], SR.upsample_bwd_replay(dyb, H, W).reshape(-1))


UP_GRID_CAP = 1 << 20
UPSAMPLE_CAP = [(17, 1024, 1024, 1, 4096, 4096, "fwd"), (17, 4096, 4096, 1, 1024, 1024, "bwd")]   # N, H, W, C, H_out, W_out, pass


@pytest.mark.parametrize("N,H,W,C,Ho,Wo,pas", UPSAMPLE_CAP, ids=["fwd-1024-4096", "bwd-4096-1024"])
def test_upsample_past_the_grid_cap(pkg, eng, N, H, W, C, Ho, Wo, pas):
    """a destination of 285 M elements at the 2^20-block cap: the last image is written on the second lap.  Images are independent,
    so images 0, 8 and 16 equal the replay on those images alone; the NaN-filled destination keeps no NaN anywhere"""
    info = pkg.upsample_bilinear_info(N, H, W, C, Ho, Wo)
    per_img = (Ho * Wo if pas == "fwd" else H * W) * C
    assert info["grid_" + pas] == UP_GRID_CAP and info["threads"] == 256
    assert (N - 1) * per_img >= UP_GRID_CAP * 256                         # the whole last image on the second lap
    src_hw = (H, W) if pas == "fwd" else (Ho, Wo)
    rng = np.random.default_rng(N + Ho)
    src = SR.bf16_bits(rng.standard_normal((N, *src_hw, C), dtype=np.float32))
    dst = nan_buf(N * per_img)
    layer = pkg.UpsampleBilinearLayer(eng, N, H, W, C, Ho, Wo)
    (layer.forward if pas == "fwd" else layer.backward)(dev_bits(src), dst)
    eng.sync()
    assert not torch.isnan(dst.view(torch.bfloat16)).any().item()
    for n in (0, 8, N - 1):
        got = host(dst[n * per_img:(n + 1) * per_img])
        want = SR.upsample_fwd_replay(src[n:n + 1], Ho, Wo) if pas == "fwd" else SR.upsample_bwd_replay(src[n:n + 1], H, W)
        assert np.array_equal(got, want.reshape(-1)), n
