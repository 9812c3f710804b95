"""Zero padding of the wide-channel convolution (pcnn_conv_wide_plan_create_padded, pcnn_conv_wide_wgrad_padded,
pcnn_conv_wide_dgrad_padded) on the GPU: exact integer results against the float64 pad-then-valid references with NaN-prefilled
outputs and an untouched NaN pad of dx, the memory pad of a pitched x never read, determinism, adjointness, the padded entry
points at padding (0, 0) bit-identical to the unpadded ones, and random operands bit-identical to the pad-copy route
(pcnn_pad_nhwc_bf16 -> the unpadded pass on the canvas -> pcnn_crop_nhwc_bf16)."""
import ctypes

import numpy as np
import pytest

import conv_ref as CR
import conv_ref_strided as CS
import test_conv_tc_gpu as G
import test_conv_wide_gpu as WG

pytestmark = pytest.mark.gpu

NAN_BF16 = G.NAN_BF16

# N, H, W, C, K, R, S, stride, pad_h, pad_w, row_pitch, image_rows (0 = dense)
CASES = [
    (2, 14, 14, 64, 64, 3, 3, 1, 1, 1, 0, 0),             # 3x3 "same"
    (2, 13, 11, 40, 24, 5, 5, 1, 2, 2, 0, 0),             # 5x5 "same", a partly filled channel chunk
    (2, 12, 12, 16, 32, 7, 7, 1, 3, 3, 0, 0),             # 7x7 "same"
    (2, 17, 15, 64, 128, 3, 3, 2, 1, 1, 0, 0),            # stride 2, pad 1: tap 0 is at row -1 (floor division)
    (2, 19, 18, 40, 24, 3, 3, 3, 2, 1, 0, 0),             # stride 3, pad_h != pad_w
    (2, 9, 10, 48, 64, 3, 2, 4, 1, 1, 0, 0),              # stride 4 > taps: phases 3 and 0 of x, dx phases without taps
    (2, 10, 21, 48, 64, 1, 7, 1, 0, 3, 0, 0),             # 1x7 padded along rows only
    (2, 26, 15, 128, 96, 3, 1, 1, 1, 0, 15 * 128 + 64, 0),  # 3x1 in a pitched layout (pad columns)
    (2, 12, 13, 320, 64, 3, 3, 1, 2, 2, 0, 0),            # "full" padding, two input-gradient channel groups
    (3, 2, 2, 64, 32, 3, 3, 1, 1, 1, 0, 0),               # H < R
    (2, 4, 5, 64, 32, 3, 3, 4, 1, 1, 0, 0),               # H = stride
    (2, 8, 8, 8, 8, 3, 3, 1, 1, 1, 0, 0),                 # C = K = 8: the row-Toeplitz plan's shape unpadded, this plan's padded
    (3, 17, 23, 64, 128, 3, 3, 2, 1, 1, 23 * 64 + 32, 20),  # stride 2 in a pitched layout (pad columns and rows)
]
MULTI = [  # the four layers of `conv_bench.py widesame`, sized so that all three passes reach their regime on 114 and 132 SMs
    (96, 56, 56, 64, 64, 3, 3, 1, 1, 1, 0, 0),
    (224, 28, 28, 128, 128, 3, 3, 1, 1, 1, 0, 0),
    (464, 14, 14, 256, 256, 3, 3, 1, 1, 1, 0, 0),
    (212, 56, 56, 64, 128, 3, 3, 2, 1, 1, 0, 0),
]


def ids(cases):
    return ["x".join(map(str, c[:7])) + f"-s{c[7]}-pad{c[8]}{c[9]}" + (f"-p{c[10]}" if c[10] else "") + (f"-r{c[11]}" if c[11] else "")
            for c in cases]


def out_size(H, W, R, S, st, ph, pw):
    return (H + 2 * ph - R) // st + 1, (W + 2 * pw - S) // st + 1


# ------------------------------------------------------------- float64 references: np.pad, then the valid convolution
def _pad(x, ph, pw):
    return np.pad(np.asarray(x, np.float64), ((0, 0), (ph, ph), (pw, pw), (0, 0)))


def fwd_ref(x, f, b, st, ph, pw):
    return CR.conv_fwd_f64(_pad(x, ph, pw), f, b, st)


def wgrad_ref(x, dy, R, S, st, ph, pw):
    return CS.conv_wgrad_f64(_pad(x, ph, pw), dy, R, S, st)


def dgrad_ref(dy, f, H, W, st, ph, pw):
    """the canvas's input gradient, cropped to the H x W image"""
    return CS.conv_dgrad_f64(dy, f, H + 2 * ph, W + 2 * pw, st)[:, ph:ph + H, pw:pw + W, :]


def regime(pkg, case, sm_count):
    """forward tiles per CTA; weight-gradient pixel blocks per unit and units; input-gradient tiles per CTA (the _padded queries)"""
    N, H, W, C, K, R, S, st, ph, pw = case[:10]
    fw = pkg.conv_wide_plan_info(N, H, W, C, K, R, S, st, padding=(ph, pw))
    b = pkg.conv_wide_bwd_info(N, H, W, C, K, R, S, st, padding=(ph, pw))
    return dict(fwd_stages=fw["stages"], fwd_min_tiles_per_cta=fw["tiles"] // min(fw["tiles"], sm_count),
                wgrad_stages=b["wgrad_stages"], wgrad_blocks_per_unit=b["wgrad_blocks_per_split"], wgrad_units=b["wgrad_units"],
                dgrad_stages=b["dgrad_stages"], dgrad_min_tiles_per_cta=b["dgrad_tiles"] // min(b["dgrad_tiles"], sm_count))


def in_regime(g, sm_count):
    return (g["fwd_min_tiles_per_cta"] > 2 * g["fwd_stages"] and g["wgrad_blocks_per_unit"] > 2 * g["wgrad_stages"]
            and g["wgrad_units"] > sm_count and g["dgrad_min_tiles_per_cta"] > 2 * g["dgrad_stages"])


# ------------------------------------------------------------------------------------------------------ running the passes
def _int_operands(rng, N, H, W, C, K, R, S, st, ph, pw):
    """x in {0..3}, dy in {-1, 0, 1}, f in {-1, 0, 1} with about 48 nonzeros per filter and per input channel: every partial sum
    is an integer below 2^24 and |y|, |dx| stay far below 256 (exact in bf16)"""
    P, Q = out_size(H, W, R, S, st, ph, pw)
    x = rng.integers(0, 4, (N, H, W, C), dtype=np.uint8)
    dy = rng.integers(-1, 2, (N, P, Q, K), dtype=np.int8)
    dens = min(0.5, 48.0 / max(R * S * C, K * R * S))
    f = (rng.random((K, R, S, C)) < dens) * rng.choice(np.array([-1, 1], np.float32), (K, R, S, C))
    return x, dy, f.astype(np.float32)


def _fwd(eng, pkg, xd, f, b, case, act=0, reps=1):
    N, H, W, C, K, R, S, st, ph, pw, pitch, rows = case
    plan = pkg.WideConvPlan(eng, N, H, W, C, K, R, S, f, b, act=act, row_pitch=pitch or W * C, image_rows=rows, stride=st,
                            padding=(ph, pw))
    assert plan.out_shape == (N,) + out_size(H, W, R, S, st, ph, pw) + (K,)
    outs = []
    for _ in range(reps):
        y = eng.to_device(np.full(plan.out_shape, NAN_BF16, np.uint16))
        plan.fwd(xd, y)
        eng.sync()
        outs.append(y.to_host())
    plan.close()
    return outs


def _wgrad(eng, xd, dyd, case):
    N, H, W, C, K, R, S, st, ph, pw, pitch, rows = case
    dw = eng.to_device(np.full((K, R, S, C), np.nan, np.float32))
    eng.conv_wide_wgrad(xd, dyd, dw, N, H, W, C, K, R, S, row_pitch=pitch or W * C, image_rows=rows, stride=st, padding=(ph, pw))
    return dw.to_host()


def _dgrad(eng, dyd, fd, case):
    """dx into a NaN-filled [N][rows][pitch] canvas: the pad must come back untouched.  Returns the bf16 bits [N, H, W, C]."""
    N, H, W, C, K, R, S, st, ph, pw, pitch, rows = case
    pitch_, rows_ = pitch or W * C, rows or H
    dxo = eng.to_device(np.full((N, rows_, pitch_), NAN_BF16, np.uint16))
    eng.conv_wide_dgrad(dyd, fd, dxo, N, H, W, C, K, R, S, row_pitch=pitch_, image_rows=rows, stride=st, padding=(ph, pw))
    out = dxo.to_host()
    assert np.all(out[:, H:, :] == NAN_BF16) and np.all(out[:, :, W * C:] == NAN_BF16)             # pad never written
    return out[:, :H, :W * C].reshape(N, H, W, C)


@pytest.mark.parametrize("case", CASES + MULTI, ids=ids(CASES + MULTI))
def test_padded_exact_integers(eng, pkg, case):
    """Integer operands: y, dw and dx bit-identical to the float64 pad-then-valid references.  Every output is prefilled with NaN,
    so every element must have been written; dx's NaN pad must be unchanged.  <y, dy> = <x, dx> = <f, dw> exactly.  The
    multi-tile cases run twice and must be bit-identical."""
    N, H, W, C, K, R, S, st, ph, pw, pitch, rows = case
    multi = case in MULTI
    if multi:
        g = regime(pkg, case, G._sm(eng))
        assert in_regime(g, G._sm(eng)), g
    reps = 2 if multi else 1
    rng = np.random.default_rng(sum(case))
    x, dy, f = _int_operands(rng, N, H, W, C, K, R, S, st, ph, pw)
    xd = eng.to_device(G._layout(G._bf16_bits(pkg, x), rows or H, pitch or W * C))
    dyd, fd = eng.to_device(G._bf16_bits(pkg, dy)), eng.to_device(f)

    ys = _fwd(eng, pkg, xd, f, None, case, reps=reps)
    y = pkg.bf16_bits_to_f32(ys[0]).astype(np.float64)
    ref = fwd_ref(x, f, None, st, ph, pw)
    assert np.abs(ref).max() < 256
    bad = y != ref                                                          # NaN (never written) is unequal too
    assert not bad.any(), ("y", np.argwhere(bad)[:5], int(bad.sum()))

    dws = [_wgrad(eng, xd, dyd, case) for _ in range(reps)]
    ref = wgrad_ref(x, dy, R, S, st, ph, pw)
    assert np.abs(ref).max() < 2 ** 24
    assert np.array_equal(dws[0], ref.astype(np.float32)), ("dw", np.argwhere(dws[0] != ref)[:5], int((dws[0] != ref).sum()))
    del xd

    dxs = [_dgrad(eng, dyd, fd, case) for _ in range(reps)]
    dx = pkg.bf16_bits_to_f32(dxs[0]).astype(np.float64)
    ref = dgrad_ref(dy, f, H, W, st, ph, pw)
    assert np.abs(ref).max() <= 256
    bad = dx != ref
    assert not bad.any(), ("dx", np.argwhere(bad)[:5], int(bad.sum()))

    a = float(np.sum(y * dy))
    b = float(np.sum(x.astype(np.float64) * dx))
    c = float(np.sum(f.astype(np.float64) * dws[0]))
    assert a == b == c, (a, b, c)
    if multi:
        assert np.array_equal(ys[0], ys[1])
        assert np.array_equal(dws[0].view(np.uint32), dws[1].view(np.uint32))
        assert np.array_equal(dxs[0], dxs[1])


@pytest.mark.parametrize("case", [c for c in CASES if c[10] or c[11]], ids=ids([c for c in CASES if c[10] or c[11]]))
def test_padded_passes_ignore_the_memory_pad(eng, pkg, case):
    """NaN in the pad columns and pad rows of a pitched x (which are not the zero padding): y and dw bit-identical to the run with
    a zero memory pad."""
    N, H, W, C, K, R, S, st, ph, pw, pitch, rows = case
    rng = np.random.default_rng(sum(case) + 1)
    P, Q = out_size(H, W, R, S, st, ph, pw)
    xb = G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C))
    f = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    dyd = eng.to_device(G._uniform_bits(pkg, rng, -1, 1, (N, P, Q, K)))
    ys, dws = [], []
    for canvas in (G._layout(xb, rows or H, pitch), G._nan_padded(xb, rows or H, pitch)):
        xd = eng.to_device(canvas)
        ys.append(_fwd(eng, pkg, xd, f, b, case)[0])
        dws.append(_wgrad(eng, xd, dyd, case))
    assert np.isfinite(pkg.bf16_bits_to_f32(ys[0])).all() and np.isfinite(dws[0]).all()
    assert np.array_equal(ys[1], ys[0]), int((ys[1] != ys[0]).sum())
    assert np.array_equal(dws[1].view(np.uint32), dws[0].view(np.uint32)), int(np.isnan(dws[1]).sum())


# ---------------------------------------------------------------------------- padding (0, 0): the unpadded entry points exactly
def _check(pkg, fn, rc):
    if rc != 0:
        raise pkg.PcnnError(fn, rc, pkg.lib().pcnn_last_error_string().decode())


def _raw_plan(eng, pkg, N, H, W, C, K, R, S, st, f, b, act):
    """a plan from pcnn_conv_wide_plan_create_padded at padding (0, 0), run by pcnn_conv_tc_fwd like WideConvPlan's"""
    plan = ctypes.c_void_p()
    b = np.ascontiguousarray(b, np.float32)
    f = np.ascontiguousarray(f, np.float32)
    _check(pkg, "pcnn_conv_wide_plan_create_padded",
              pkg.lib().pcnn_conv_wide_plan_create_padded(eng.ctx, N, H, W, C, K, R, S, st, 0, 0, W * C, 0, act, f.ctypes.data,
                                                          b.ctypes.data, ctypes.byref(plan)))
    return plan


@pytest.mark.parametrize("case", WG.WIDE_CASES, ids=WG.WIDE_IDS)
def test_padded_entry_points_at_zero_padding_are_the_unpadded_ones(eng, pkg, case):
    """Random operands, sigmoid: the three _padded entry points called with padding (0, 0) give the bits of the unpadded ones."""
    N, H, W, C, K, R, S, st = case
    P, Q = out_size(H, W, R, S, st, 0, 0)
    rng = np.random.default_rng(sum(case) + 2)
    xb = G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    xd, fd = eng.to_device(xb), eng.to_device(f)
    dyd = eng.to_device(G._uniform_bits(pkg, rng, -1, 1, (N, P, Q, K)))
    L = pkg.lib()

    y0 = WG._run(eng, pkg, xb.reshape(N, H, W * C), f, b, N, H, W, C, K, R, S, st, act=1)[0]
    plan = _raw_plan(eng, pkg, N, H, W, C, K, R, S, st, f, b, 1)
    try:
        y1 = eng.to_device(np.full((N, P, Q, K), NAN_BF16, np.uint16))
        _check(pkg, "pcnn_conv_tc_fwd", L.pcnn_conv_tc_fwd(eng.ctx, plan, ctypes.c_void_p(xd.ptr), ctypes.c_void_p(y1.ptr)))
        eng.sync()
    finally:
        L.pcnn_conv_tc_plan_destroy(eng.ctx, plan)
    assert np.array_equal(y1.to_host(), y0)

    dw0, dw1 = eng.array((K, R, S, C)), eng.to_device(np.full((K, R, S, C), np.nan, np.float32))
    eng.conv_wide_wgrad(xd, dyd, dw0, N, H, W, C, K, R, S, stride=st)
    _check(pkg, "pcnn_conv_wide_wgrad_padded", L.pcnn_conv_wide_wgrad_padded(eng.ctx, xd.ptr, dyd.ptr, dw1.ptr, N, H, W, C, K, R, S, st,
                                                                             0, 0, W * C, 0))
    assert np.array_equal(dw1.to_host().view(np.uint32), dw0.to_host().view(np.uint32))

    dx0, dx1 = eng.array((N, H, W * C), np.uint16), eng.to_device(np.full((N, H, W * C), NAN_BF16, np.uint16))
    eng.conv_wide_dgrad(dyd, fd, dx0, N, H, W, C, K, R, S, stride=st)
    _check(pkg, "pcnn_conv_wide_dgrad_padded", L.pcnn_conv_wide_dgrad_padded(eng.ctx, dyd.ptr, fd.ptr, dx1.ptr, N, H, W, C, K, R, S, st,
                                                                             0, 0, W * C, 0))
    assert np.array_equal(dx1.to_host(), dx0.to_host())


# --------------------------------------------------------------------------------------------------- the pad-copy route
def _canvas_in_wide_domain(pkg, case):
    N, H, W, C, K, R, S, st, ph, pw = case[:10]
    try:
        pkg.conv_wide_plan_info(N, H + 2 * ph, W + 2 * pw, C, K, R, S, st)
        return True
    except pkg.PcnnError:
        return False


ROUTE = [c for c in CASES + MULTI if c[:10] != (2, 8, 8, 8, 8, 3, 3, 1, 1, 1)]   # C = K = 8: its canvas is the row-Toeplitz plan's


@pytest.mark.parametrize("case", ROUTE, ids=ids(ROUTE))
def test_padded_passes_are_the_pad_copy_route(eng, pkg, case):
    """Random operands (bias and sigmoid on the forward): y, dw and dx bit-identical to pcnn_pad_nhwc_bf16 -> the unpadded wide
    pass on the canvas (-> pcnn_crop_nhwc_bf16 for dx).  Forward and weight gradient issue the same tiles, operand boxes and
    MMAs; the input gradient adds the same taps in the same (i, j, 64-filter chunk) order into every element."""
    N, H, W, C, K, R, S, st, ph, pw, pitch, rows = case
    assert _canvas_in_wide_domain(pkg, case)
    Hc, Wc = H + 2 * ph, W + 2 * pw
    P, Q = out_size(H, W, R, S, st, ph, pw)
    rng = np.random.default_rng(sum(case) + 3)
    xb = G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C))
    dyb = G._uniform_bits(pkg, rng, -1, 1, (N, P, Q, K))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    dyd, fd = eng.to_device(dyb), eng.to_device(f)
    canvas = eng.to_device(np.full((N, Hc, Wc * C), NAN_BF16, np.uint16))
    eng.pad_nhwc(eng.to_device(xb), canvas, N, H, W, C, ph, pw)
    xd = eng.to_device(G._layout(xb, rows or H, pitch or W * C))
    full = (N, Hc, Wc, C, K, R, S, st, 0, 0, 0, 0)

    y = _fwd(eng, pkg, xd, f, b, case, act=1)[0]
    y_route = _fwd(eng, pkg, canvas, f, b, full, act=1)[0]
    assert np.array_equal(y, y_route), ("y", int((y != y_route).sum()))

    dw, dw_route = _wgrad(eng, xd, dyd, case), _wgrad(eng, canvas, dyd, full)
    assert np.isfinite(dw).all()
    assert np.array_equal(dw.view(np.uint32), dw_route.view(np.uint32)), ("dw", int((dw != dw_route).sum()))
    del xd, canvas

    dx = _dgrad(eng, dyd, fd, case)
    dxc = eng.array((N, Hc, Wc * C), np.uint16)
    eng.conv_wide_dgrad(dyd, fd, dxc, N, Hc, Wc, C, K, R, S, stride=st)
    dx_route = eng.to_device(np.full((N, H, W * C), NAN_BF16, np.uint16))
    eng.crop_nhwc(dxc, dx_route, N, H, W, C, ph, pw)
    dx_route = dx_route.to_host().reshape(N, H, W, C)
    assert np.array_equal(dx, dx_route), ("dx", int((dx != dx_route).sum()))


def test_padded_gradients_name_themselves_in_refusals(eng, pkg):
    """A padding outside 0..R-1 is refused by both gradients, naming the called function and the rule."""
    N, H, W, C, K, R, S = 2, 14, 14, 64, 64, 3, 3
    xd = eng.to_device(np.zeros((N, H, W * C), np.uint16))
    dyd = eng.to_device(np.zeros((N, H, W, K), np.uint16))
    fd = eng.to_device(np.zeros((K, R, S, C), np.float32))
    with pytest.raises(pkg.PcnnError, match=r"pcnn_conv_wide_wgrad_padded: padding \(3, 1\).*pad_h <= R - 1") as e:
        eng.conv_wide_wgrad(xd, dyd, eng.array((K, R, S, C)), N, H, W, C, K, R, S, padding=(3, 1))
    assert e.value.code == -1
    with pytest.raises(pkg.PcnnError, match=r"pcnn_conv_wide_dgrad_padded: H = 3, W = 14 with padding \(1, 1\) at stride 4") as e:
        eng.conv_wide_dgrad(dyd, fd, xd, N, 3, W, C, K, R, S, stride=4, padding=(1, 1))
    assert e.value.code == -1
