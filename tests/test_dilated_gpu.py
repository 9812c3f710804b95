"""Dilated convolution on the GPU (pcnn_conv_wide_plan_create_dilated, pcnn_conv_wide_wgrad_dilated, pcnn_conv_wide_dgrad_dilated,
pcnn_dwconv_plan_create_dilated and the layers over them).

Wide passes: exact integer results against the float64 references of dilated_ref.py (pinned to torch by test_dilated_cpu.py) with
NaN-prefilled outputs, dx's pad untouched, NaN in x's memory pad changing no bit, reruns bit-identical and <y, dy> = <x, dx> =
<f, dw> exactly; random operands within the bound models of test_conv_wide_gpu.py / test_conv_wide_bwd_gpu.py; and, where the
window's extent is at most 7, the padded passes with the filters zero-inserted to E x E give the same results.  Depthwise: y and
dx bit-identical to the float32 replays with +-0, +-Inf and NaN, dw exact on integers and within the n_acc bound otherwise, every
refusal.  Layers: one step against float64, and the forward after set_params, SGD and AdamW bit-identical to a fresh plan."""
import numpy as np
import pytest

import dilated_ref as D
import test_conv_tc_gpu as G
import test_conv_wide_bwd_gpu as WB
import test_dilated_cpu as DC
import test_dwconv_gpu as DG

pytestmark = pytest.mark.gpu

NAN_BF16 = G.NAN_BF16

# N, H, W, C, K, R, S, stride, (pad_h, pad_w), (dil_h, dil_w), row_pitch, image_rows (0 = dense)
CASES = [
    (2, 15, 14, 64, 64, 3, 3, 1, (2, 2), (2, 2), 0, 0),         # stride 1, d 2 "same"
    (2, 16, 17, 40, 24, 3, 3, 1, (3, 1), (3, 3), 0, 0),         # stride 1, d 3, pad_h != pad_w, a partial channel chunk
    (2, 20, 19, 64, 32, 3, 3, 1, (6, 6), (6, 6), 0, 0),         # stride 1, d 6 "same"
    (2, 19, 18, 64, 64, 3, 3, 2, (2, 2), (2, 2), 0, 0),         # stride 2, d 2: g = 2, dx phases with odd a + pad have no taps
    (2, 21, 20, 48, 64, 3, 3, 2, (3, 3), (3, 3), 0, 0),         # stride 2, d 3: coprime
    (2, 22, 23, 64, 32, 3, 3, 3, (2, 1), (2, 2), 0, 0),         # stride 3, d 2
    (2, 25, 26, 64, 64, 3, 3, 4, (4, 4), (4, 4), 0, 0),         # stride 4, d 4: g = 4, one dx row phase in four has taps
    (2, 11, 30, 48, 64, 1, 7, 1, (0, 9), (1, 3), 0, 0),         # 1x7 taps at dilation (1, 3)
    (2, 13, 12, 64, 64, 1, 3, 2, (0, 2), (5, 2), 0, 0),         # R = 1 with a row dilation that no tap uses
    (2, 14, 13, 320, 64, 3, 3, 1, (2, 2), (2, 2), 0, 0),        # C = 320: two input-gradient channel groups
    (2, 17, 15, 64, 128, 3, 3, 2, (2, 2), (2, 2), 15 * 64 + 32, 20),   # pitched x: pad columns and pad rows
    (2, 12, 12, 64, 32, 3, 3, 1, (0, 0), (3, 3), 0, 0),         # no padding
]
BENCH = [c[:8] + ((c[8], c[8]), (c[9], c[9]), 0, 0) for c in DC.BENCH if c[9] > 1]


def ids(cases):
    return [f"{c[1]}x{c[2]}x{c[3]}-{c[4]}-{c[5]}x{c[6]}-s{c[7]}-p{c[8][0]}{c[8][1]}-d{c[9][0]}{c[9][1]}" + ("-pitched" if c[10] else "")
            + (f"-n{c[0]}" if c[0] > 2 else "") for c in cases]


def _out(case):
    N, H, W, C, K, R, S, st, pad, dil = case[:10]
    return D.out_size(H, W, R, S, st, pad, dil)


def _fwd(eng, pkg, xd, f, b, case, act=0, reps=1):
    N, H, W, C, K, R, S, st, pad, dil, pitch, rows = case
    plan = pkg.WideConvPlan(eng, N, H, W, C, K, R, S, f, b, act=act, row_pitch=pitch or W * C, image_rows=rows, stride=st,
                            padding=pad, dilation=dil)
    assert plan.out_shape == (N,) + _out(case) + (K,)
    outs = []
    for _ in range(reps):
        y = eng.to_device(np.full(plan.out_shape, NAN_BF16, np.uint16))
        plan.fwd(xd, y)
        eng.sync()
        outs.append(y.to_host())
    plan.close()
    return outs


def _wgrad(eng, xd, dyd, case):
    N, H, W, C, K, R, S, st, pad, dil, pitch, rows = case
    dw = eng.to_device(np.full((K, R, S, C), np.nan, np.float32))
    eng.conv_wide_wgrad(xd, dyd, dw, N, H, W, C, K, R, S, row_pitch=pitch or W * C, image_rows=rows, stride=st, padding=pad, dilation=dil)
    return dw.to_host()


def _dgrad(eng, dyd, fd, case):
    """dx into a NaN-filled [N][rows][pitch] canvas, whose pad must come back untouched; the bf16 bits [N, H, W, C]"""
    N, H, W, C, K, R, S, st, pad, dil, pitch, rows = case
    pitch_, rows_ = pitch or W * C, rows or H
    dxo = eng.to_device(np.full((N, rows_, pitch_), NAN_BF16, np.uint16))
    eng.conv_wide_dgrad(dyd, fd, dxo, N, H, W, C, K, R, S, row_pitch=pitch_, image_rows=rows, stride=st, padding=pad, dilation=dil)
    out = dxo.to_host()
    assert np.all(out[:, H:, :] == NAN_BF16) and np.all(out[:, :, W * C:] == NAN_BF16)
    return out[:, :H, :W * C].reshape(N, H, W, C)


def _int_operands(rng, case):
    """x in {0..3}, dy and f in {-1, 0, 1}, about 48 nonzero filter taps per filter and input channel: every partial sum is an
    integer below 2^24 and |y|, |dx| stay below 256 (exact in bf16)"""
    N, H, W, C, K, R, S = case[:7]
    P, Q = _out(case)
    x = rng.integers(0, 4, (N, H, W, C), dtype=np.uint8)
    dy = rng.integers(-1, 2, (N, P, Q, K), dtype=np.int8)
    dens = min(0.5, 48.0 / max(R * S * C, K * R * S))
    f = (rng.random((K, R, S, C)) < dens) * rng.choice(np.array([-1, 1], np.float32), (K, R, S, C))
    return x, dy, f.astype(np.float32)


@pytest.mark.parametrize("case", CASES + BENCH, ids=ids(CASES + BENCH))
def test_dilated_exact_integers(eng, pkg, case):
    """Integer operands: y, dw and dx bit-identical to the float64 references; every output prefilled with NaN and fully written;
    dx's NaN pad unchanged; <y, dy> = <x, dx> = <f, dw> exactly; a rerun bit-identical.  The benchmark shapes first check that
    they run in their regime on this GPU."""
    N, H, W, C, K, R, S, st, pad, dil, pitch, rows = case
    if case in BENCH:
        g = DC.bench_regime(pkg, case[:8] + (pad[0], dil[0]), G._sm(eng))
        assert all(g.values()), g
    rng = np.random.default_rng(sum(case[:8]) + dil[0])
    x, dy, f = _int_operands(rng, case)
    xd = eng.to_device(G._layout(G._bf16_bits(pkg, x), rows or H, pitch or W * C))
    dyd, fd = eng.to_device(G._bf16_bits(pkg, dy)), eng.to_device(f)

    ys = _fwd(eng, pkg, xd, f, None, case, reps=2)
    y = pkg.bf16_bits_to_f32(ys[0]).astype(np.float64)
    ref = D.fwd_f64(x, f, None, st, pad, dil)
    assert np.abs(ref).max() < 256
    bad = y != ref
    assert not bad.any(), ("y", np.argwhere(bad)[:5], int(bad.sum()))

    dws = [_wgrad(eng, xd, dyd, case) for _ in range(2)]
    ref = D.wgrad_f64(x, dy, R, S, st, pad, dil)
    assert np.abs(ref).max() < 2 ** 24
    assert np.array_equal(dws[0], ref.astype(np.float32)), ("dw", np.argwhere(dws[0] != ref)[:5], int((dws[0] != ref).sum()))
    del xd

    dxs = [_dgrad(eng, dyd, fd, case) for _ in range(2)]
    dx = pkg.bf16_bits_to_f32(dxs[0]).astype(np.float64)
    ref = D.dgrad_f64(dy, f, H, W, st, pad, dil)
    assert np.abs(ref).max() <= 256
    bad = dx != ref
    assert not bad.any(), ("dx", np.argwhere(bad)[:5], int(bad.sum()))

    a = float(np.sum(y * dy))
    b = float(np.sum(x.astype(np.float64) * dx))
    c = float(np.sum(f.astype(np.float64) * dws[0]))
    assert a == b == c, (a, b, c)
    assert np.array_equal(ys[0], ys[1])
    assert np.array_equal(dws[0].view(np.uint32), dws[1].view(np.uint32))
    assert np.array_equal(dxs[0], dxs[1])


PITCHED = [c for c in CASES if c[10]]


@pytest.mark.parametrize("case", PITCHED, ids=ids(PITCHED))
def test_dilated_passes_ignore_the_memory_pad(eng, pkg, case):
    """NaN in the pad columns and rows of a pitched x changes no bit of y or dw"""
    N, H, W, C, K, R, S, st, pad, dil, pitch, rows = case
    rng = np.random.default_rng(sum(case[:8]) + 1)
    P, Q = _out(case)
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
    assert np.array_equal(ys[1], ys[0])
    assert np.array_equal(dws[1].view(np.uint32), dws[0].view(np.uint32))


@pytest.mark.parametrize("case", CASES, ids=ids(CASES))
def test_dilated_random_within_bounds(eng, pkg, case):
    """Random operands: y (bias, no activation), dw and dx within the error models of the wide passes (test_conv_wide_gpu.py,
    test_conv_wide_bwd_gpu.py): |z - ref| <= 2 (T/16 + 1) 2^-23 M then one bf16 rounding for y, T = R S C; 2 n_acc 2^-23 sum|x dy|
    with n_acc = 8 blocks per unit + splits for dw; e = 2 R S ceil(K/16) 2^-23 sum|dy f| then one bf16 rounding for dx"""
    N, H, W, C, K, R, S, st, pad, dil, pitch, rows = case
    P, Q = _out(case)
    rng = np.random.default_rng(sum(case[:8]) + 3)
    xb = G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C))
    dyb = G._uniform_bits(pkg, rng, -1, 1, (N, P, Q, K))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    x, dyf = pkg.bf16_bits_to_f32(xb).astype(np.float64), pkg.bf16_bits_to_f32(dyb).astype(np.float64)
    xd = eng.to_device(G._layout(xb, rows or H, pitch or W * C))
    dyd = eng.to_device(dyb)

    y = pkg.bf16_bits_to_f32(_fwd(eng, pkg, xd, f, b, case)[0]).astype(np.float64)
    ref = D.fwd_f64(x, f, b, st, pad, dil)
    mag = D.fwd_f64(x, np.abs(f), np.abs(b), st, pad, dil)
    e = 2 * (R * S * C / 16 + 1) * 2.0 ** -23 * mag
    assert WB._worst_ratio(np.abs(y - ref), e + 2.0 ** -8 * (np.abs(ref) + e)) <= 1.0

    info = pkg.conv_wide_bwd_info(N, H, W, C, K, R, S, st, pitch or None, rows, padding=pad, dilation=dil)
    n_acc = 8 * (info["wgrad_blocks_per_split"] + 1) + info["wgrad_splits"]
    dw = _wgrad(eng, xd, dyd, case).astype(np.float64)
    ref = D.wgrad_f64(x, dyf, R, S, st, pad, dil)
    mag = D.wgrad_f64(x, np.abs(dyf), R, S, st, pad, dil)
    assert WB._worst_ratio(np.abs(dw - ref), 2 * n_acc * 2.0 ** -23 * mag) <= 1.0

    dx = pkg.bf16_bits_to_f32(_dgrad(eng, dyd, eng.to_device(f), case)).astype(np.float64)
    ref = D.dgrad_f64(dyf, f, H, W, st, pad, dil)
    e = 2 * R * S * -(-K // 16) * 2.0 ** -23 * D.dgrad_f64(np.abs(dyf), np.abs(f), H, W, st, pad, dil)
    assert WB._worst_ratio(np.abs(dx - ref), e + 2.0 ** -8 * (np.abs(ref) + e)) <= 1.0


CROSS = [c for c in CASES if (c[5] - 1) * c[9][0] + 1 <= 7 and (c[6] - 1) * c[9][1] + 1 <= 7]


@pytest.mark.parametrize("case", CROSS, ids=ids(CROSS))
def test_dilated_passes_equal_padded_passes_on_zero_inserted_filters(eng, pkg, case):
    """Without torch: where E <= 7, the padded (undilated) passes with the filters zero-inserted to E_h x E_w give dw bit-identical
    at the dilated taps (and +0 between them), and y and dx equal to the dilated passes' (a different sign of a zero is reported:
    the extra taps add exact zeros after the same nonzero terms, so no other difference can occur)"""
    N, H, W, C, K, R, S, st, pad, dil, pitch, rows = case
    P, Q = _out(case)
    rng = np.random.default_rng(sum(case[:8]) + 5)
    xb = G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C))
    dyb = G._uniform_bits(pkg, rng, -1, 1, (N, P, Q, K))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    fz = D.zero_inserted(f, dil)
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    Re, Se = fz.shape[1:3]
    zcase = (N, H, W, C, K, Re, Se, st, pad, (1, 1), pitch, rows)
    xd, dyd = eng.to_device(G._layout(xb, rows or H, pitch or W * C)), eng.to_device(dyb)

    y, yz = _fwd(eng, pkg, xd, f, b, case)[0], _fwd(eng, pkg, xd, fz, b, zcase)[0]
    diff = y != yz
    zero = ((y & 0x7FFF) == 0) & ((yz & 0x7FFF) == 0)
    print(f"{case}: y differs in {int(diff.sum())} elements, {int((diff & zero).sum())} of them by the sign of a zero")
    assert not (diff & ~zero).any()

    dw, dwz = _wgrad(eng, xd, dyd, case), _wgrad(eng, xd, dyd, zcase)
    assert np.array_equal(dwz[:, ::dil[0], ::dil[1], :].view(np.uint32), dw.view(np.uint32))

    fd, fzd = eng.to_device(f), eng.to_device(fz)
    dx, dxz = _dgrad(eng, dyd, fd, case), _dgrad(eng, dyd, fzd, zcase)
    diff = dx != dxz
    zero = ((dx & 0x7FFF) == 0) & ((dxz & 0x7FFF) == 0)
    print(f"{case}: dx differs in {int(diff.sum())} elements, {int((diff & zero).sum())} of them by the sign of a zero")
    assert not (diff & ~zero).any()


# ----------------------------------------------------------------------------------------------------------------- depthwise
DW_CASES = [  # id, N, H, W, C, R, S, stride, pad, dilation
    ("c8-3x3s1-d2", 2, 13, 12, 8, 3, 3, 1, (2, 2), (2, 2)),
    ("c16-3x3s2-d2", 2, 14, 15, 16, 3, 3, 2, (2, 2), (2, 2)),
    ("c5-5x5s1-d2", 2, 17, 16, 5, 5, 5, 1, (4, 4), (2, 2)),
    ("c32-3x3s1-d6", 2, 20, 19, 32, 3, 3, 1, (6, 6), (6, 6)),
    ("c3-3x3s3-d23", 2, 11, 13, 3, 3, 3, 3, (1, 3), (2, 3)),
    ("c8-1x7s1-d13", 2, 9, 25, 8, 1, 7, 1, (0, 3), (1, 3)),
    ("c24-7x7s4-d2", 2, 16, 16, 24, 7, 7, 4, (5, 6), (2, 2)),
    ("c144-3x3s1-d3-nopad", 2, 9, 10, 144, 3, 3, 1, (0, 0), (3, 3)),
    ("c320-3x3s2-d4", 2, 15, 14, 320, 3, 3, 2, (4, 4), (4, 4)),
    ("c32-3x3s1-d6-deeplab", 32, 14, 14, 32, 3, 3, 1, (6, 6), (6, 6)),
    ("c144-3x3s1-d2-bench", 128, 56, 56, 144, 3, 3, 1, (2, 2), (2, 2)),
]


@pytest.mark.parametrize("case", DW_CASES, ids=[c[0] for c in DW_CASES])
def test_depthwise_dilated_passes(eng, pkg, case):
    """y (bias, ReLU) and dx bit-identical to the float32 replays with +-0, +-Inf and NaN in x, w and dy; nothing past any output
    written; dw exact on integer operands and within 2 n_acc 2^-24 sum|dy x| on random ones"""
    _, N, H, W, C, R, S, st, pad, dil = case
    rng = np.random.default_rng(N * H + C + dil[0])
    P, Q = D.out_size(H, W, R, S, st, pad, dil)
    bf, f32 = pkg.f32_to_bf16_bits, pkg.bf16_bits_to_f32
    x_bits = bf(DG.special(rng, (N, H, W, C)))
    w = f32(bf(DG.special(rng, (C, R, S))))
    b = rng.standard_normal(C).astype(np.float32)
    dy_bits = bf(DG.special(rng, (N, P, Q, C)))
    plan = pkg.DepthwiseConvPlan(eng, N, H, W, C, R, S, w, b, act=3, stride=st, padding=pad, dilation=dil)
    assert plan.out_shape == (N, P, Q, C)
    y = DG.run_fwd(eng, plan, x_bits, plan.out_shape)
    assert DG.same_or_nan(y, bf(D.dw_fwd(f32(x_bits), w, b, st, pad, dil, act=3)))
    dx = DG.run_dgrad(eng, plan, dy_bits, (N, H, W, C))
    assert DG.same_or_nan(dx, bf(D.dw_dgrad(f32(dy_bits), w, H, W, st, pad, dil)))
    plan.close()

    xi = rng.integers(-3, 4, (N, H, W, C)).astype(np.float32)
    dyi = rng.integers(-2, 3, (N, P, Q, C)).astype(np.float32)
    plan = pkg.DepthwiseConvPlan(eng, N, H, W, C, R, S, w * 0, None, stride=st, padding=pad, dilation=dil)
    dw = DG.run_wgrad(eng, plan, bf(xi), bf(dyi), C, R, S)
    assert np.array_equal(dw.astype(np.float64), D.dw_wgrad_f64(xi, dyi, R, S, st, pad, dil))
    xr, dyr = f32(bf(rng.standard_normal((N, H, W, C)).astype(np.float32))), f32(bf(rng.standard_normal((N, P, Q, C)).astype(np.float32)))
    dw = DG.run_wgrad(eng, plan, bf(xr), bf(dyr), C, R, S).astype(np.float64)
    n_acc = pkg.dwconv_info(N, H, W, C, R, S, st, pad, dil)["n_acc"]
    ref, mag = D.dw_wgrad_f64(xr, dyr, R, S, st, pad, dil), D.dw_wgrad_f64(np.abs(xr), np.abs(dyr), R, S, st, pad, dil)
    assert np.all(np.abs(dw - ref) <= 2 * n_acc * DG.U * mag)
    plan.close()


def test_depthwise_dilated_refusals(eng, pkg):
    """each domain rule of pcnn_dwconv_plan_create_dilated refused with its text, naming the call"""
    w = np.zeros((8, 3, 3), np.float32)
    fn = "pcnn_dwconv_plan_create_dilated"
    for kw, pat in [(dict(dilation=(0, 1)), r"dilation \(0, 1\): 1 <= dil_h, dil_w <= 256"),
                    (dict(dilation=(2, 257)), r"dilation \(2, 257\)"),
                    (dict(padding=(5, 1), dilation=(2, 2)), r"padding \(5, 1\) for a 3x3 filter at dilation \(2, 2\): 0 <= pad_h <= dil_h \(R - 1\)"),
                    (dict(padding=(-1, 1), dilation=(2, 2)), r"padding \(-1, 1\)"),
                    (dict(H=4, padding=(0, 0), dilation=(2, 2)), r"a 3x3 filter at dilation \(2, 2\) does not fit the 4x9 image padded by \(0, 0\): H \+ 2 pad_h >= dil_h \(R - 1\) \+ 1"),
                    (dict(stride=5, dilation=(2, 2)), r"stride 5"),
                    (dict(N=0, dilation=(2, 2)), r"N = 0")]:
        args = dict(N=2, H=9, W=9, stride=1, padding=(1, 1))
        args.update(kw)
        with pytest.raises(pkg.PcnnError, match=fn + ": " + pat):
            pkg.DepthwiseConvPlan(eng, args["N"], args["H"], args["W"], 8, 3, 3, w, stride=args["stride"], padding=args["padding"],
                                  dilation=args.get("dilation", (1, 1)))


# -------------------------------------------------------------------------------------------------------------------- layers
def test_dilated_conv_layer_step(eng, pkg):
    """One step of a dilated ConvLayer (bias, ReLU) against float64 on integer operands: y, db, dw and dx exact; after set_params,
    SGD and AdamW the forward is bit-identical to a fresh plan made from the new master"""
    N, H, W, C, K, R, S, st, pad, dil = 4, 14, 14, 32, 32, 3, 3, 1, (2, 2), (2, 2)
    rng = np.random.default_rng(11)
    f = ((rng.random((K, R, S, C)) < 0.15) * rng.choice(np.array([-1.0, 1.0], np.float32), (K, R, S, C))).astype(np.float32)
    b = rng.integers(-2, 3, K).astype(np.float32)
    layer = pkg.ConvLayer(eng, N, H, W, C, K, R, S, f, b, act=3, stride=st, padding=pad, dilation=dil)
    assert layer.family == "wide" and layer.out_shape == (N, H, W, K)
    x = rng.integers(0, 4, (N, H, W, C)).astype(np.float32)
    dy = rng.integers(-1, 2, (N, H, W, K)).astype(np.float32)
    xd = eng.to_device(pkg.f32_to_bf16_bits(x))
    y = eng.array(layer.out_shape, np.uint16)
    layer.forward(xd, y)
    dx = eng.array((N, H, W, C), np.uint16)
    layer.backward(y, eng.to_device(pkg.f32_to_bf16_bits(dy)), dx)
    eng.sync()
    pre = D.fwd_f64(x, f, b, st, pad, dil)
    assert np.array_equal(pkg.bf16_bits_to_f32(y.to_host()).astype(np.float64), np.maximum(pre, 0))
    dpre = np.where(pre > 0, dy, 0.0)
    assert np.array_equal(layer.db.to_host().astype(np.float64), dpre.sum(axis=(0, 1, 2)))
    assert np.array_equal(layer.dw.to_host().astype(np.float64), D.wgrad_f64(x, dpre, R, S, st, pad, dil))
    assert np.array_equal(pkg.bf16_bits_to_f32(dx.to_host()).reshape(N, H, W, C).astype(np.float64), D.dgrad_f64(dpre, f, H, W, st, pad, dil))
    _refresh_checks(eng, pkg, layer, xd, lambda wm, bm: pkg.WideConvPlan(eng, N, H, W, C, K, R, S, wm, bm, act=3, stride=st, padding=pad,
                                                                          dilation=dil))
    layer.close()


def test_dilated_depthwise_layer_step(eng, pkg):
    """One step of a dilated DepthwiseConvLayer (bias, ReLU) against float64 on integer operands; the same refresh checks"""
    N, H, W, C, R, S, st, pad, dil = 4, 14, 14, 32, 3, 3, 1, (6, 6), (6, 6)
    rng = np.random.default_rng(12)
    w = rng.integers(-2, 3, (C, R, S)).astype(np.float32)
    b = rng.integers(-2, 3, C).astype(np.float32)
    layer = pkg.DepthwiseConvLayer(eng, N, H, W, C, R, S, w, b, act=3, stride=st, padding=pad, dilation=dil)
    assert layer.out_shape == (N, H, W, C)
    x = rng.integers(-3, 4, (N, H, W, C)).astype(np.float32)
    dy = rng.integers(-1, 2, (N, H, W, C)).astype(np.float32)
    xd = eng.to_device(pkg.f32_to_bf16_bits(x))
    y = eng.array(layer.out_shape, np.uint16)
    layer.forward(xd, y)
    dx = eng.array((N, H, W, C), np.uint16)
    layer.backward(y, eng.to_device(pkg.f32_to_bf16_bits(dy)), dx)
    eng.sync()
    pre = D.dw_fwd(x.astype(np.float64), w, b, st, pad, dil)
    assert np.array_equal(pkg.bf16_bits_to_f32(y.to_host()).astype(np.float64), np.maximum(pre, 0))
    dpre = np.where(pre > 0, dy, 0.0)
    assert np.array_equal(layer.db.to_host().astype(np.float64), dpre.sum(axis=(0, 1, 2)))
    assert np.array_equal(layer.dw.to_host().astype(np.float64), D.dw_wgrad_f64(x, dpre, R, S, st, pad, dil))
    assert np.array_equal(pkg.bf16_bits_to_f32(dx.to_host()).astype(np.float64), D.dw_dgrad(dpre, w.astype(np.float64), H, W, st, pad, dil))
    _refresh_checks(eng, pkg, layer, xd, lambda wm, bm: pkg.DepthwiseConvPlan(eng, N, H, W, C, R, S, wm, bm, act=3, stride=st, padding=pad,
                                                                               dilation=dil))
    layer.close()


def _refresh_checks(eng, pkg, layer, xd, fresh_plan):
    """after set_params (new random masters), then SGD and AdamW steps on the current gradients, the layer's forward equals that of
    a fresh plan built from its master"""
    rng = np.random.default_rng(13)

    def same_as_fresh():
        eng.sync()
        wm, bm = layer.params()
        fresh = fresh_plan(wm, bm)
        y0, y1 = eng.array(layer.out_shape, np.uint16), eng.array(layer.out_shape, np.uint16)
        layer.plan.fwd(xd, y0)
        fresh.fwd(xd, y1)
        eng.sync()
        assert np.array_equal(y0.to_host(), y1.to_host())
        fresh.close()

    wm, bm = layer.params()
    nw = eng.to_device(rng.standard_normal(wm.shape).astype(np.float32) * 0.1)
    nb = eng.to_device(rng.standard_normal(bm.shape).astype(np.float32) * 0.1)
    layer.plan.set_params(nw, nb)
    eng.sync()
    fresh = fresh_plan(nw.to_host(), nb.to_host())
    y0, y1 = eng.array(layer.out_shape, np.uint16), eng.array(layer.out_shape, np.uint16)
    layer.plan.fwd(xd, y0)
    fresh.fwd(xd, y1)
    eng.sync()
    assert np.array_equal(y0.to_host(), y1.to_host())
    fresh.close()
    layer.plan.set_params(layer.filt, layer.bias)
    for opt in (pkg.SGD(eng, [layer], momentum=0.9, weight_decay=1e-2), pkg.AdamW(eng, [layer], weight_decay=0.05)):
        for _ in range(2):
            opt.step(0.05)
        same_as_fresh()
        opt.close()
