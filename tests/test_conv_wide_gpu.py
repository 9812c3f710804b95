"""The wide-channel convolution forward (pcnn_conv_wide_plan_create, csrc/conv_wide_tc.cu) on the GPU against the float64
reference conv_ref.conv_fwd_f64: exact integer results with NaN-prefilled outputs, random operands with sigmoid within a
stated bound, NaN row padding, "same" padding, adjointness with the input gradient, determinism, and the unchanged refusal of
ConvPlan next to a WideConvPlan that runs the same shape."""
import numpy as np
import pytest

import conv_ref as CR
import conv_ref_strided as CS
import test_conv_tc_gpu as G

pytestmark = pytest.mark.gpu

NAN_BF16 = G.NAN_BF16

WIDE_CASES = [  # N, H, W, C, K, R, S, stride: small shapes covering the rules, one or a few tiles per CTA
    (3, 14, 14, 16, 8, 3, 3, 1),        # 12x12 outputs (8x16 blocks issue 256 pixels for 144), K = 8 (MMA width 16)
    (2, 20, 23, 40, 64, 5, 5, 1),       # C = 40: a partly filled 64-channel chunk; ragged blocks
    (2, 13, 13, 64, 120, 7, 7, 1),      # 7x7 outputs, 7x7 taps, K = 120 (MMA width 128, filters 120..127 zero-filled)
    (2, 16, 19, 128, 256, 1, 7, 1),     # 1x7 taps, K = 256
    (2, 17, 15, 256, 64, 3, 1, 2),      # 3x1 taps, stride 2, four chunks
    (3, 30, 29, 64, 64, 3, 3, 4),       # stride 4 (gaps between windows)
    (2, 9, 200, 40, 16, 1, 1, 1),       # 1x1 on a long row: 1 x 128 pixel blocks
    (2, 23, 22, 24, 32, 2, 2, 3),       # 2x2 taps, stride 3, (W - S) % stride != 0
    (2, 21, 21, 16, 64, 5, 5, 2),       # 5x5, stride 2
]
WIDE_IDS = ["x".join(map(str, c[:7])) + f"-s{c[7]}" for c in WIDE_CASES]

WIDE_MULTI = [  # N, H, W, C, K, R, S, stride: the five layers of `conv_bench.py wide`, at > 2 x stages tiles per CTA on 114 and 132 SMs
    (96, 56, 56, 64, 64, 3, 3, 1),
    (224, 28, 28, 128, 128, 3, 3, 1),
    (464, 14, 14, 256, 256, 3, 3, 1),   # small images: 256 pixels issued per 144 computed
    (36, 56, 56, 64, 256, 1, 1, 1),
    (212, 56, 56, 64, 128, 3, 3, 2),
]
MULTI_IDS = ["x".join(map(str, c[:7])) + f"-s{c[7]}" for c in WIDE_MULTI]


def wide_regime(pkg, N, H, W, C, K, R, S, stride, sm_count):
    pl = pkg.conv_wide_plan_info(N, H, W, C, K, R, S, stride)
    grid = min(pl["tiles"], sm_count)
    return dict(pl, grid=grid, min_tiles_per_cta=pl["tiles"] // grid)


def _int_operands(rng, N, H, W, C, K, R, S):
    """x in {0..3}; each filter has at most 64 nonzero taps, each +-1; bias in {-4..4}: every partial sum is an integer below
    2^24 and |y| <= 3 * 64 + 4 < 256, exact in bf16"""
    x = rng.integers(0, 4, (N, H, W, C), dtype=np.uint8)
    f = np.zeros((K, R * S * C), np.float32)
    nz = min(64, R * S * C)
    for k in range(K):
        f[k, rng.choice(R * S * C, nz, replace=False)] = rng.choice(np.array([-1, 1], np.float32), nz)
    b = rng.integers(-4, 5, K).astype(np.float32)
    return x, f.reshape(K, R, S, C), b


def _run(eng, pkg, canvas, f, b, N, H, W, C, K, R, S, stride, act=0, pitch=None, rows=0, reps=1):
    plan = pkg.WideConvPlan(eng, N, H, W, C, K, R, S, f, b, act=act, row_pitch=pitch, image_rows=rows, stride=stride)
    xd = eng.to_device(canvas)
    outs = []
    for _ in range(reps):
        y = eng.to_device(np.full(plan.out_shape, NAN_BF16, np.uint16))
        plan.fwd(xd, y)
        eng.sync()
        outs.append(y.to_host())
    plan.close()
    return outs


def _check_exact(pkg, x, f, b, stride, got):
    for n0 in range(0, x.shape[0], 16):
        ref = CR.conv_fwd_f64(x[n0:n0 + 16], f, b, stride)
        assert np.array_equal(ref, np.round(ref)) and np.abs(ref).max() <= 256
        g = pkg.bf16_bits_to_f32(got[n0:n0 + 16])
        bad = g != ref.astype(np.float32)                   # NaN (an element never written) is unequal too
        assert not bad.any(), (n0, np.argwhere(bad)[:5], int(bad.sum()))


@pytest.mark.parametrize("case", WIDE_CASES + WIDE_MULTI, ids=WIDE_IDS + MULTI_IDS)
def test_wide_forward_exact_integers(eng, pkg, case):
    """Sparse small-integer operands: bit-identical to the float64 reference, every output element written (y prefilled with
    NaN).  The multi-tile cases run twice and must be bit-identical (determinism)."""
    N, H, W, C, K, R, S, st = case
    multi = case in WIDE_MULTI
    if multi:
        g = wide_regime(pkg, N, H, W, C, K, R, S, st, G._sm(eng))
        assert g["min_tiles_per_cta"] > 2 * g["stages"], g
    rng = np.random.default_rng(sum(case))
    x, f, b = _int_operands(rng, N, H, W, C, K, R, S)
    pitch = W * C
    outs = _run(eng, pkg, G._layout(G._bf16_bits(pkg, x), H, pitch), f, b, N, H, W, C, K, R, S, st, reps=2 if multi else 1)
    _check_exact(pkg, x, f, b, st, outs[0])
    if multi:
        assert np.array_equal(outs[0], outs[1])


@pytest.mark.parametrize("case", WIDE_CASES + WIDE_MULTI, ids=WIDE_IDS + MULTI_IDS)
def test_wide_forward_random_with_sigmoid(eng, pkg, case):
    """x ~ U[0,1), f ~ U[-0.5,0.5), bias ~ U[-0.5,0.5), bf16-rounded, sigmoid epilogue; float64 reference on the same operands.

    Error model: the pre-activation z is a sum of T = R*S*C products x*f, each exact in fp32 (bf16 operands).  wgmma adds them
    in steps of 16 products into one fp32 accumulator: T/16 accumulator updates plus one for the bias.  Every update rounds once,
    by at most 2^-23 of a running value that never exceeds M = sum |x*f| + |bias| (one ulp, which covers a truncating
    accumulator; a step's 16 products are reduced inside the tensor core, which may round once more: c = 2).  So
        |z_got - z| <= c * (T/16 + 1) * 2^-23 * M.
    The sigmoid (slope <= 1/4) is tanh.approx-based, within a_act = 5e-4 absolute, and the bf16 result is rounded once, by at most
    half an ulp, 2^-8 of its magnitude.  With a = a_act + (1/4) * c * (T/16 + 1) * 2^-23 * M:
        |y_got - y| <= a + 2^-8 (|y| + a).
    The worst ratio of |y_got - y| to the bound is printed.  Multi-tile cases check their first and last 16 images."""
    N, H, W, C, K, R, S, st = case
    rng = np.random.default_rng(sum(case) + 7)
    xb = G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    got = _run(eng, pkg, G._layout(xb, H, W * C), f, b, N, H, W, C, K, R, S, st, act=1)[0]
    T = R * S * C
    worst = 0.0
    for n0 in sorted({0, max(0, N - 16)}):
        xs = pkg.bf16_bits_to_f32(xb[n0:n0 + 16])
        z = CR.conv_fwd_f64(xs, f, b, st)
        mag = CR.conv_fwd_f64(xs, np.abs(f), None, st) + np.abs(b)          # x >= 0: sum |x * f| + |bias|
        ref = 1.0 / (1.0 + np.exp(-z))
        dz = 2 * (T / 16 + 1) * 2.0 ** -23 * mag
        a = 5e-4 + 0.25 * dz
        bound = a + 2.0 ** -8 * (np.abs(ref) + a)
        ratio = np.abs(pkg.bf16_bits_to_f32(got[n0:n0 + 16]) - ref) / bound
        worst = max(worst, float(np.max(ratio)))
    print(f"wide fwd {case}: worst |got - ref| / bound = {worst:.3e}")
    assert worst <= 1.0, worst


@pytest.mark.parametrize("case", [(64, 30, 30, 64, 64, 3, 3, 1, 30 * 64 + 16, 33),
                                  (48, 31, 29, 40, 120, 3, 3, 2, 29 * 40 + 8, 34),
                                  (32, 16, 16, 256, 256, 1, 1, 1, 16 * 256 + 64, 17)],
                         ids=["c64_s1", "c40_s2", "c256_1x1"])
def test_wide_forward_ignores_row_padding(eng, pkg, case):
    """NaN in the pad columns (pitch > W*C) and the pad rows (image_rows > H) of x: the output bits equal the zero-padded run."""
    N, H, W, C, K, R, S, st, pitch, rows = case
    rng = np.random.default_rng(sum(case))
    xb = G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C))
    f = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    zero = _run(eng, pkg, G._layout(xb, rows, pitch), f, b, N, H, W, C, K, R, S, st, pitch=pitch, rows=rows)[0]
    nan = _run(eng, pkg, G._nan_padded(xb, rows, pitch), f, b, N, H, W, C, K, R, S, st, pitch=pitch, rows=rows)[0]
    assert np.isfinite(pkg.bf16_bits_to_f32(zero)).all()
    assert np.array_equal(nan, zero), int((nan != zero).sum())


def test_wide_same_convolution_through_pad(eng, pkg):
    """A "same" 3x3 convolution: pcnn_pad_nhwc_bf16 into the tight canvas, then the wide plan, against the float64 reference on
    np.pad (exact integers)."""
    N, H, W, C, K, R, S = 6, 19, 21, 48, 64, 3, 3
    rng = np.random.default_rng(11)
    x, f, b = _int_operands(rng, N, H, W, C, K, R, S)
    src = eng.to_device(G._bf16_bits(pkg, x))
    canvas = eng.to_device(np.full((N, H + 2, (W + 2) * C), NAN_BF16, np.uint16))
    eng.pad_nhwc(src, canvas, N, H, W, C, 1, 1)
    plan = pkg.WideConvPlan(eng, N, H + 2, W + 2, C, K, R, S, f, b)
    assert plan.out_shape == (N, H, W, K)
    y = eng.to_device(np.full(plan.out_shape, NAN_BF16, np.uint16))
    plan.fwd(canvas, y)
    eng.sync()
    plan.close()
    ref = CR.conv_fwd_f64(np.pad(x, ((0, 0), (1, 1), (1, 1), (0, 0))), f, b)
    assert np.array_equal(pkg.bf16_bits_to_f32(y.to_host()), ref.astype(np.float32))


@pytest.mark.parametrize("shape", [(2, 15, 17, 16, 24, 3, 3, 2), (3, 12, 11, 40, 16, 3, 3, 1), (2, 14, 13, 8, 32, 5, 5, 3)])
def test_wide_forward_is_the_adjoint_of_the_input_gradient(eng, pkg, shape):
    """Integer x, f, dy: <y, dy> = <x, dx> exactly, with dx from pcnn_conv_dgrad_strided on the FMA reference path (every shape).
    The new forward is the transpose of the input gradient the library already defines for this layer."""
    N, H, W, C, K, R, S, st = shape
    rng = np.random.default_rng(sum(shape))
    P, Q = CS.out_size(H, W, R, S, st)
    x, f, _ = _int_operands(rng, N, H, W, C, K, R, S)
    dy = rng.integers(-1, 2, (N, P, Q, K)).astype(np.float32)
    y = _run(eng, pkg, G._layout(G._bf16_bits(pkg, x), H, W * C), f, None, N, H, W, C, K, R, S, st)[0]
    dx = eng.to_device(np.full((N, H, W * C), NAN_BF16, np.uint16))
    eng.conv_bwd_select(reference=True)
    try:
        eng.conv_dgrad(eng.to_device(G._bf16_bits(pkg, dy)), eng.to_device(f), dx, N, H, W, C, K, R, S, stride=st)
        eng.sync()
    finally:
        eng.conv_bwd_select(reference=False)
    dxf = pkg.bf16_bits_to_f32(dx.to_host()).reshape(N, H, W, C).astype(np.float64)
    dx_ref = CS.conv_dgrad_f64(dy, f, H, W, st)
    assert np.abs(dx_ref).max() <= 256 and np.array_equal(dxf, dx_ref)          # exact in bf16
    yf = pkg.bf16_bits_to_f32(y).astype(np.float64)
    lhs, rhs = float(np.sum(yf * dy)), float(np.sum(x.astype(np.float64) * dxf))
    assert lhs == rhs, (lhs, rhs)


def test_conv_plan_still_refuses_what_the_wide_plan_runs(eng, pkg):
    """ConvPlan refuses C = 64 (3x3) as before; WideConvPlan runs the same shape through the same pcnn_conv_tc_fwd."""
    N, H, W, C, K, R, S = 2, 32, 32, 64, 64, 3, 3
    f = np.zeros(K * R * S * C, np.float32)
    with pytest.raises(pkg.PcnnError):
        pkg.ConvPlan(eng, N, H, W, C, K, R, S, f)
    rng = np.random.default_rng(3)
    x, f, b = _int_operands(rng, N, H, W, C, K, R, S)
    got = _run(eng, pkg, G._bf16_bits(pkg, x).reshape(N, H, W * C), f, b, N, H, W, C, K, R, S, 1)[0]
    _check_exact(pkg, x, f, b, 1, got)
