"""The gradients of the wide-channel forward (pcnn_conv_wide_wgrad / pcnn_conv_wide_dgrad, csrc/conv_wide_bwd_tc.cu) on the GPU
against the float64 references of tests/conv_ref_strided.py: exact integer results with NaN-prefilled outputs and an untouched
NaN pad, random operands within stated bounds, adjointness with WideConvPlan, agreement with the FMA-pipe reference kernels,
NaN row padding of x, determinism, and the unchanged refusals of the existing backward entry points."""
import numpy as np
import pytest

import conv_ref as CR
import conv_ref_strided as CS
import test_conv_tc_gpu as G
import test_conv_wide_gpu as WG

pytestmark = pytest.mark.gpu

NAN_BF16 = G.NAN_BF16

# N, H, W, C, K, R, S, stride, row_pitch, image_rows (0 = dense)
CASES = [c + (0, 0) for c in WG.WIDE_CASES] + [
    (2, 12, 13, 320, 64, 3, 3, 1, 0, 0),                 # C = 320: two input-gradient channel groups (192 + 128)
    (2, 19, 18, 40, 24, 2, 3, 4, 0, 0),                  # stride 4 > R, S: uncovered rows and columns, phases without taps
    (3, 17, 23, 64, 128, 3, 3, 3, 23 * 64 + 32, 20),     # stride 3, padded layout
    (2, 21, 20, 48, 64, 1, 7, 2, 20 * 48 + 8, 23),       # 1x7 taps at stride 2, padded layout
    (2, 26, 15, 128, 96, 3, 1, 1, 15 * 128 + 64, 0),     # 3x1 taps, pad columns only
]
MULTI = [  # the five layers of `conv_bench.py widebwd`, sized so that both passes reach their regime on 114 and 132 SMs
    (96, 56, 56, 64, 64, 3, 3, 1, 0, 0),
    (224, 28, 28, 128, 128, 3, 3, 1, 0, 0),
    (464, 14, 14, 256, 256, 3, 3, 1, 0, 0),
    (152, 56, 56, 64, 256, 1, 1, 1, 0, 0),              # one row block: warpgroup 1 idles, the pixel ranges carry the parallelism
    (128, 56, 56, 64, 128, 3, 3, 2, 0, 0),
]


def _ids(cases):
    return ["x".join(map(str, c[:7])) + f"-s{c[7]}" + (f"-p{c[8]}" if c[8] else "") + (f"-r{c[9]}" if c[9] else "") for c in cases]


def regime(pkg, case8, sm_count):
    """the weight gradient's work units and pixel blocks per unit, the input gradient's tiles per CTA"""
    N, H, W, C, K, R, S, st = case8
    b = pkg.conv_wide_bwd_info(N, H, W, C, K, R, S, st)
    blocks = pkg.conv_wide_plan_info(N, H, W, C, K, R, S, st)["tiles"]
    w = dict(stages=b["wgrad_stages"], units=b["wgrad_units"], splits=b["wgrad_splits"], blocks_per_unit=b["wgrad_blocks_per_split"],
             max_blocks_per_unit=-(-blocks // b["wgrad_splits"]))
    grid = min(b["dgrad_tiles"], sm_count)
    d = dict(stages=b["dgrad_stages"], tiles=b["dgrad_tiles"], grid=grid, min_tiles_per_cta=b["dgrad_tiles"] // grid)
    return w, d


def _assert_regime(pkg, eng, case):
    sm = G._sm(eng)
    w, d = regime(pkg, case[:8], sm)
    assert w["blocks_per_unit"] > 2 * w["stages"] and w["units"] > sm, w
    assert d["min_tiles_per_cta"] > 2 * d["stages"], d
    return w, d


def _worst_ratio(err, bound):
    """max of err / bound; where the bound is 0 (an output no product reaches) the result must be exact"""
    ok = bound > 0
    r = np.where(ok, err / np.where(ok, bound, 1.0), np.where(err == 0, 0.0, np.inf))
    return float(r.max())


def _int_operands(rng, N, H, W, C, K, R, S, st):
    """x in {0..3}, dy in {-1, 0, 1}, f in {-1, 0, 1} with about 48 nonzeros per filter and per input channel: every partial sum
    is an integer below 2^24, |y| and |dx| stay far below 256 (exact in bf16)"""
    P, Q = CS.out_size(H, W, R, S, st)
    x = rng.integers(0, 4, (N, H, W, C), dtype=np.uint8)
    dy = rng.integers(-1, 2, (N, P, Q, K), dtype=np.int8)
    dens = min(0.5, 48.0 / max(R * S * C, K * R * S))
    f = (rng.random((K, R, S, C)) < dens) * rng.choice(np.array([-1, 1], np.float32), (K, R, S, C))
    return x, dy, f.astype(np.float32)


def _dgrad(eng, pkg, dyd, fd, case, reference=False):
    """dx into a NaN-filled [N][rows][pitch] canvas: the pad must come back untouched.  Returns the bf16 bits [N, H, W, C]."""
    N, H, W, C, K, R, S, st, pitch, rows = case
    pitch_, rows_ = pitch or W * C, rows or H
    dxo = eng.to_device(np.full((N, rows_, pitch_), NAN_BF16, np.uint16))
    if reference:
        eng.conv_dgrad(dyd, fd, dxo, N, H, W, C, K, R, S, row_pitch=pitch_, image_rows=rows, stride=st)
    else:
        eng.conv_wide_dgrad(dyd, fd, dxo, N, H, W, C, K, R, S, row_pitch=pitch_, image_rows=rows, stride=st)
    out = dxo.to_host()
    assert np.all(out[:, H:, :] == NAN_BF16) and np.all(out[:, :, W * C:] == NAN_BF16)             # pad never written
    return out[:, :H, :W * C].reshape(N, H, W, C)


def _wgrad(eng, xd, dyd, case):
    N, H, W, C, K, R, S, st, pitch, rows = case
    dw = eng.to_device(np.full((K, R, S, C), np.nan, np.float32))
    eng.conv_wide_wgrad(xd, dyd, dw, N, H, W, C, K, R, S, row_pitch=pitch or W * C, image_rows=rows, stride=st)
    return dw.to_host()


@pytest.mark.parametrize("case", CASES + MULTI, ids=_ids(CASES + MULTI))
def test_wide_backward_exact_integers(eng, pkg, case):
    """Integer operands: dw and dx bit-identical to the float64 references.  dw and dx are prefilled with NaN, so every element,
    the zeros of dx rows and columns no window covers included, must have been written; dx's NaN pad must be unchanged.  The
    multi-tile cases run twice and must be bit-identical."""
    N, H, W, C, K, R, S, st, pitch, rows = case
    multi = case in MULTI
    if multi:
        _assert_regime(pkg, eng, case)
    rng = np.random.default_rng(sum(case))
    x, dy, f = _int_operands(rng, N, H, W, C, K, R, S, st)
    xd = eng.to_device(G._layout(G._bf16_bits(pkg, x), rows or H, pitch or W * C))
    dyd, fd = eng.to_device(G._bf16_bits(pkg, dy)), eng.to_device(f)
    dws = [_wgrad(eng, xd, dyd, case) for _ in range(2 if multi else 1)]
    ref = CS.conv_wgrad_f64(x, dy, R, S, st)
    assert np.abs(ref).max() < 2 ** 24
    assert np.array_equal(dws[0], ref.astype(np.float32)), (np.argwhere(dws[0] != ref)[:5], int((dws[0] != ref).sum()))
    del xd
    dxs = [_dgrad(eng, pkg, dyd, fd, case) for _ in range(2 if multi else 1)]
    got = pkg.bf16_bits_to_f32(dxs[0])
    for n0 in range(0, N, 16):
        ref = CS.conv_dgrad_f64(dy[n0:n0 + 16], f, H, W, st)
        assert np.abs(ref).max() <= 256
        bad = got[n0:n0 + 16] != ref.astype(np.float32)                    # NaN (never written) is unequal too
        assert not bad.any(), (n0, np.argwhere(bad)[:5], int(bad.sum()))
    if multi:
        assert np.array_equal(dws[0].view(np.uint32), dws[1].view(np.uint32))
        assert np.array_equal(dxs[0], dxs[1])


@pytest.mark.parametrize("case", CASES + MULTI, ids=_ids(CASES + MULTI))
def test_wide_backward_random(eng, pkg, case):
    """x ~ U[0,1), dy ~ U[-1,1), f ~ U[-0.5,0.5), bf16-rounded; float64 references on the same operands.

    Weight gradient: an element is a sum of N*P*Q products x*dy, each exact in fp32.  A work unit adds them into one register
    accumulator 16 pixels per wgmma: 8 updates per pixel block, at most max_blocks_per_unit blocks; the slot reduction adds one
    partial per pixel range (`splits` additions, fixed order).  Every update rounds once, by at most 2^-23 of a running value
    that never exceeds sum|x*dy| (one ulp, which covers a truncating accumulator); the tensor core's own reduction of a step's 16
    products may round once more: c = 2.  So
        |got - ref| <= 2 * n_acc * 2^-23 * sum|x*dy|,   n_acc = 8 * max_blocks_per_unit + splits.
    Input gradient: a sum of at most T = R*S*ceil(K/16) wgmma steps into one fp32 accumulator, with the same per-step model,
    e = 2 * T * 2^-23 * sum|dy*f|, then one bf16 rounding (half an ulp, <= 2^-8 of the magnitude):
        |got - ref| <= e + 2^-8 (|ref| + e).
    The worst ratios to the bounds are printed.  Multi-tile cases check dx on their first and last 16 images."""
    N, H, W, C, K, R, S, st, pitch, rows = case
    P, Q = CS.out_size(H, W, R, S, st)
    w_reg, _ = regime(pkg, case[:8], G._sm(eng))
    rng = np.random.default_rng(sum(case) + 3)
    xb = G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C))
    dyb = G._uniform_bits(pkg, rng, -1, 1, (N, P, Q, K))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    dyd = eng.to_device(dyb)
    x, dyf, dya = G._Decoded(pkg, xb), G._Decoded(pkg, dyb), G._Decoded(pkg, dyb, absolute=True)
    got = _wgrad(eng, eng.to_device(G._layout(xb, rows or H, pitch or W * C)), dyd, case).astype(np.float64)
    ref, mag = CS.conv_wgrad_f64(x, dyf, R, S, st), CS.conv_wgrad_f64(x, dya, R, S, st)      # x >= 0: sum |x * dy|
    n_acc = 8 * w_reg["max_blocks_per_unit"] + w_reg["splits"]
    wr = _worst_ratio(np.abs(got - ref), 2 * n_acc * 2.0 ** -23 * mag)
    dx = pkg.bf16_bits_to_f32(_dgrad(eng, pkg, dyd, eng.to_device(f), case))
    T = R * S * -(-K // 16)
    dr = 0.0
    for n0 in sorted({0, max(0, N - 16)} if case in MULTI else range(0, N, 16)):
        ref = CS.conv_dgrad_f64(dyf[n0:n0 + 16], f, H, W, st)
        e = 2 * T * 2.0 ** -23 * CS.conv_dgrad_f64(dya[n0:n0 + 16], np.abs(f), H, W, st)
        dr = max(dr, _worst_ratio(np.abs(dx[n0:n0 + 16] - ref), e + 2.0 ** -8 * (np.abs(ref) + e)))
    print(f"wide bwd {case}: wgrad n_acc {n_acc}, worst ratio {wr:.3e}; dgrad worst ratio {dr:.3e}")
    assert wr <= 1.0 and dr <= 1.0, (wr, dr)


ADJOINT = [(2, 15, 17, 16, 24, 3, 3, 2), (3, 12, 11, 40, 16, 3, 3, 1), (2, 14, 13, 8, 32, 5, 5, 3), (2, 19, 18, 40, 24, 2, 3, 4),
           (2, 12, 13, 320, 64, 3, 3, 1)]


@pytest.mark.parametrize("shape", ADJOINT, ids=["x".join(map(str, c)) for c in ADJOINT])
def test_wide_backward_is_the_adjoint_of_the_wide_forward(eng, pkg, shape):
    """Integer x, f, dy; y from WideConvPlan on the same x and f (no bias): <y, dy> = <x, dx> = <f, dw> exactly."""
    N, H, W, C, K, R, S, st = shape
    rng = np.random.default_rng(sum(shape))
    x, dy, f = _int_operands(rng, N, H, W, C, K, R, S, st)
    try:
        pkg.conv_tc_plan_info(N, H, W, C, K, R, S, st)
        pytest.fail("the row-Toeplitz plan takes this shape")
    except pkg.PcnnError:
        pass
    xd = eng.to_device(G._bf16_bits(pkg, x).reshape(N, H, W * C))
    y = pkg.bf16_bits_to_f32(WG._run(eng, pkg, G._bf16_bits(pkg, x).reshape(N, H, W * C), f, None, N, H, W, C, K, R, S, st)[0])
    assert np.array_equal(y, CR.conv_fwd_f64(x, f, None, st))                  # exact: |y| < 256
    case = (N, H, W, C, K, R, S, st, 0, 0)
    dyd = eng.to_device(G._bf16_bits(pkg, dy))
    dw = _wgrad(eng, xd, dyd, case).astype(np.float64)
    dx = pkg.bf16_bits_to_f32(_dgrad(eng, pkg, dyd, eng.to_device(f), case)).astype(np.float64)
    a = float(np.sum(y.astype(np.float64) * dy))
    b = float(np.sum(x.astype(np.float64) * dx))
    c = float(np.sum(f.astype(np.float64) * dw))
    assert a == b == c, (a, b, c)


@pytest.mark.parametrize("case", CASES + MULTI, ids=_ids(CASES + MULTI))
def test_wide_backward_against_the_fma_reference_kernels(eng, pkg, case):
    """Integer operands: dx bit-identical to pcnn_conv_dgrad_strided on the FMA-pipe reference path for every case; dw the same
    wherever that path's weight gradient runs (K*R*S*C <= 5120)."""
    N, H, W, C, K, R, S, st, pitch, rows = case
    rng = np.random.default_rng(sum(case) + 5)
    x, dy, f = _int_operands(rng, N, H, W, C, K, R, S, st)
    xd = eng.to_device(G._layout(G._bf16_bits(pkg, x), rows or H, pitch or W * C))
    dyd, fd = eng.to_device(G._bf16_bits(pkg, dy)), eng.to_device(f)
    dw, dx = _wgrad(eng, xd, dyd, case), _dgrad(eng, pkg, dyd, fd, case)
    eng.conv_bwd_select(reference=True)
    try:
        dx_ref = _dgrad(eng, pkg, dyd, fd, case, reference=True)
        if K * R * S * C <= 5120:
            dw_ref = eng.array((K, R, S, C))
            eng.conv_wgrad(xd, dyd, dw_ref, N, H, W, C, K, R, S, row_pitch=pitch or W * C, image_rows=rows, stride=st)
            assert np.array_equal(dw.view(np.uint32), dw_ref.to_host().view(np.uint32))
    finally:
        eng.conv_bwd_select(reference=False)
    assert np.array_equal(dx, dx_ref), int((dx != dx_ref).sum())


@pytest.mark.parametrize("case", [c for c in CASES if c[8] or c[9]] + [(64, 30, 30, 64, 64, 3, 3, 1, 30 * 64 + 16, 33)],
                         ids=_ids([c for c in CASES if c[8] or c[9]]) + ["c64_multi"])
def test_wide_weight_gradient_ignores_row_padding(eng, pkg, case):
    """NaN in the pad columns and pad rows of x: dw is bit-identical to the zero-padded run."""
    N, H, W, C, K, R, S, st, pitch, rows = case
    rng = np.random.default_rng(sum(case))
    P, Q = CS.out_size(H, W, R, S, st)
    xb = G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C))
    dyd = eng.to_device(G._uniform_bits(pkg, rng, -1, 1, (N, P, Q, K)))
    out = [_wgrad(eng, eng.to_device(canvas), dyd, case) for canvas in (G._layout(xb, rows or H, pitch), G._nan_padded(xb, rows or H, pitch))]
    assert np.isfinite(out[0]).all()
    assert np.array_equal(out[1].view(np.uint32), out[0].view(np.uint32)), int(np.isnan(out[1]).sum())


def test_existing_backward_entry_points_still_refuse_what_the_wide_ones_run(eng, pkg):
    """The tensor-core pcnn_conv_wgrad / pcnn_conv_dgrad refuse a wide shape naming pcnn_conv_bwd_select, as before; the new
    entry points run that shape, and refuse a shape outside the wide domain naming themselves."""
    case = (2, 32, 32, 64, 64, 3, 3, 1, 0, 0)
    N, H, W, C, K, R, S = case[:7]
    rng = np.random.default_rng(4)
    x, dy, f = _int_operands(rng, N, H, W, C, K, R, S, 1)
    xd, dyd, fd = eng.to_device(G._bf16_bits(pkg, x)), eng.to_device(G._bf16_bits(pkg, dy)), eng.to_device(f)
    with pytest.raises(pkg.PcnnError, match="pcnn_conv_bwd_select"):
        eng.conv_wgrad(xd, dyd, eng.array((K, R, S, C)), N, H, W, C, K, R, S)
    with pytest.raises(pkg.PcnnError, match="pcnn_conv_bwd_select"):
        eng.conv_dgrad(dyd, fd, eng.array((N, H, W * C), np.uint16), N, H, W, C, K, R, S)
    assert np.array_equal(_wgrad(eng, xd, dyd, case), CS.conv_wgrad_f64(x, dy, R, S).astype(np.float32))
    assert np.array_equal(pkg.bf16_bits_to_f32(_dgrad(eng, pkg, dyd, fd, case)), CS.conv_dgrad_f64(dy, f, H, W).astype(np.float32))
    for fn in ("wgrad", "dgrad"):
        with pytest.raises(pkg.PcnnError, match=f"pcnn_conv_wide_{fn}: C = 36 channels") as e:
            getattr(eng, f"conv_wide_{fn}")(xd if fn == "wgrad" else dyd, dyd if fn == "wgrad" else fd, eng.array(64), 2, 28, 28, 36, 64, 3, 3)
        assert e.value.code == -1
