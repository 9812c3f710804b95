"""GPU tests of the backward passes of strided convolutions (pcnn_conv_wgrad_strided / pcnn_conv_dgrad_strided): the wgmma
kernels of csrc/conv_wgrad_tc.cu and csrc/conv_dgrad_tc.cu with a window step of 2..4, at the sizes of BWD_STRIDED_MULTI
(many tiles per CTA, shares longer than the stage ring), against the float64 references of tests/conv_ref_strided.py, the
strided forward they are the gradient of, and the FMA-pipe reference kernels."""
import importlib

import numpy as np
import pytest

import conv_ref as CR
import conv_ref_strided as CS
import test_conv_tc_gpu as G

pytestmark = pytest.mark.gpu

MULTI = CS.BWD_STRIDED_MULTI
IDS = ["x".join(map(str, c[:7])) + f"-s{c[7]}" + (f"-p{c[8]}" if c[8] else "") + (f"-r{c[9]}" if c[9] else "") for c in MULTI]
NAN_BF16 = G.NAN_BF16


def _regime(pkg, eng, N, H, W, C, K, R, S, st):
    sm = G._sm(eng)
    w, d = CS.wgrad_regime(pkg, N, H, W, C, K, R, S, sm, st), CS.dgrad_regime(pkg, N, H, W, C, K, R, S, sm, st)
    if w is not None:
        assert w["min_tiles_per_cta"] > 2 * w["stages"], w
    assert d is not None and d["max_units_per_share"] > d["stages"] and d["shares_crossing_images"] > 0, d
    return w, d


def _operands(rng, N, H, W, C, K, R, S, st, xmax):
    P, Q = CS.out_size(H, W, R, S, st)
    x = rng.integers(0, xmax + 1, (N, H, W, C), dtype=np.uint8)
    dy = rng.integers(-1, 2, (N, P, Q, K), dtype=np.int8)                       # dy in {-1, 0, 1}
    f = rng.choice(np.array([-1, 0, 0, 1], np.float32), (K, R, S, C))          # f in {-1, 0, 1}, half zeros
    return x, dy, f


def _dgrad(eng, dyd, f, N, H, W, C, K, R, S, st, pitch, rows):
    """dx into a NaN-filled [N][rows][pitch] canvas; the pad must come back untouched.  Returns float32 [N, H, W, C]."""
    pitch_, rows_ = pitch or W * C, rows or H
    dxo = eng.to_device(np.full((N, rows_, pitch_), NAN_BF16, np.uint16))
    eng.conv_dgrad(dyd, eng.to_device(f), dxo, N, H, W, C, K, R, S, row_pitch=pitch, image_rows=rows, stride=st)
    out = dxo.to_host()
    assert np.all(out[:, H:, :] == NAN_BF16) and np.all(out[:, :, W * C:] == NAN_BF16)             # pad never written
    return out[:, :H, :W * C].reshape(N, H, W, C)


@pytest.mark.parametrize("case", MULTI, ids=IDS)
def test_strided_backward_exact_at_many_tiles_per_cta(eng, pkg, case):
    """Integer operands: dw and dx bit-identical to the float64 references.  Outputs are NaN-prefilled, so every in-image dx
    element, the zeros of rows and columns no window covers included, must have been written."""
    N, H, W, C, K, R, S, st, pitch, rows = case
    w_reg, _ = _regime(pkg, eng, N, H, W, C, K, R, S, st)
    P, Q = CS.out_size(H, W, R, S, st)
    pitch_, rows_ = pitch or W * C, rows or H
    rng = np.random.default_rng(sum(case))
    xmax = 3 if 3 * N * P * Q < 2 ** 24 else 1
    assert xmax * N * P * Q < 2 ** 24
    x, dy, f = _operands(rng, N, H, W, C, K, R, S, st, xmax)
    dyd = eng.to_device(G._bf16_bits(pkg, dy))
    xd = eng.to_device(G._layout(G._bf16_bits(pkg, x), rows_, pitch_))
    if w_reg is not None:
        ref = CS.conv_wgrad_f64(x, dy, R, S, st).astype(np.float32)
        dw = eng.to_device(np.full((K, R, S, C), np.nan, np.float32))
        eng.conv_wgrad(xd, dyd, dw, N, H, W, C, K, R, S, row_pitch=pitch, image_rows=rows, stride=st)
        got = dw.to_host()
        assert np.array_equal(got, ref), (np.argwhere(got != ref)[:5], int((got != ref).sum()))
        eng.conv_wgrad(xd, dyd, dw, N, H, W, C, K, R, S, row_pitch=pitch, image_rows=rows, stride=st)
        assert np.array_equal(dw.to_host().view(np.uint32), got.view(np.uint32))                  # reruns are bit-identical
    else:
        with pytest.raises(pkg.PcnnError, match="pcnn_conv_bwd_select"):
            eng.conv_wgrad(xd, dyd, eng.array((K, R, S, C)), N, H, W, C, K, R, S, row_pitch=pitch, image_rows=rows, stride=st)
    del xd
    got = pkg.bf16_bits_to_f32(_dgrad(eng, dyd, f, N, H, W, C, K, R, S, st, pitch, rows))
    for n0 in range(0, N, 16):
        ref = CS.conv_dgrad_f64(dy[n0:n0 + 16], f, H, W, st)
        assert np.array_equal(ref, np.round(ref)) and np.abs(ref).max() <= 256
        bad = got[n0:n0 + 16] != ref.astype(np.float32)
        assert not bad.any(), (n0, np.argwhere(bad)[:5], int(bad.sum()))


@pytest.mark.parametrize("case", MULTI, ids=IDS)
def test_strided_backward_random_at_many_tiles_per_cta(eng, pkg, case):
    """x ~ U[0,1), dy ~ U[-1,1), f ~ U[-0.5,0.5), bf16-rounded.  Input gradient |d| <= 2^-8 |ref| + 1e-3; weight gradient
    within the accumulation model of test_conv_tc_gpu.test_backward_random_at_many_tiles_per_cta:
        |got - ref| <= 2 * n_acc * 2^-23 * sum|dy*x|,   n_acc = tiles_per_cta * PC/16 + RB + slots."""
    N, H, W, C, K, R, S, st, pitch, rows = case
    w_reg, _ = _regime(pkg, eng, N, H, W, C, K, R, S, st)
    P, Q = CS.out_size(H, W, R, S, st)
    pitch_, rows_ = pitch or W * C, rows or H
    rng = np.random.default_rng(sum(case) + 3)
    xb = G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C))
    dyb = G._uniform_bits(pkg, rng, -1, 1, (N, P, Q, K))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    dyd = eng.to_device(dyb)
    x, dyf = G._Decoded(pkg, xb), G._Decoded(pkg, dyb)
    if w_reg is not None:
        xd = eng.to_device(G._layout(xb, rows_, pitch_))
        dw = eng.array((K, R, S, C))
        eng.conv_wgrad(xd, dyd, dw, N, H, W, C, K, R, S, row_pitch=pitch, image_rows=rows, stride=st)
        got = dw.to_host().astype(np.float64)
        del xd
        ref = CS.conv_wgrad_f64(x, dyf, R, S, st)
        mag = CS.conv_wgrad_f64(x, G._Decoded(pkg, dyb, absolute=True), R, S, st)
        n_acc = w_reg["max_tiles_per_cta"] * w_reg["PC"] // 16 + w_reg["RB"] + w_reg["grid"]
        ratio = float(np.max(np.abs(got - ref) / (2 * n_acc * 2.0 ** -23 * mag)))
        print(f"strided wgrad {case}: n_acc {n_acc}, worst |got - ref| / bound = {ratio:.3e}")
        assert ratio <= 1.0, ratio
    got = pkg.bf16_bits_to_f32(_dgrad(eng, dyd, f, N, H, W, C, K, R, S, st, pitch, rows))
    worst = 0.0
    for n0 in range(0, N, 16):
        ref = CS.conv_dgrad_f64(dyf[n0:n0 + 16], f, H, W, st)
        err = np.abs(got[n0:n0 + 16] - ref)
        worst = max(worst, float(np.max(err / (2.0 ** -8 * np.abs(ref) + 1e-3))))
    print(f"strided dgrad {case}: worst |got - ref| / bound = {worst:.3e}")
    assert worst <= 1.0, worst


ADJOINT = [  # N, H, W, C, K, R, S, stride, image_rows (a multiple of the stride, as the forward plan requires)
    (4, 64, 40, 3, 64, 3, 3, 2, 64),
    (6, 28, 28, 1, 16, 5, 5, 2, 28),
    (3, 33, 30, 2, 32, 3, 3, 3, 36),
    (4, 42, 40, 1, 64, 3, 3, 4, 44),
]


@pytest.mark.parametrize("case", ADJOINT, ids=["x".join(map(str, c[:8])) for c in ADJOINT])
def test_strided_backward_is_the_adjoint_of_the_strided_forward(eng, pkg, case):
    """Integer x, f, dy; y = the strided forward plan (no bias, no activation).  <y, dy> = <x, dx> = <f, dw> exactly in float64:
    the backward passes are the gradients of the forward that already exists."""
    N, H, W, C, K, R, S, st, rows = case
    pitch = (W * C + 7) // 8 * 8
    rng = np.random.default_rng(sum(case))
    x = rng.integers(0, 4, (N, H, W, C), dtype=np.uint8)
    f = rng.integers(-1, 2, (K, R, S, C)).astype(np.float32)
    P, Q = CS.out_size(H, W, R, S, st)
    dy = rng.integers(-2, 3, (N, P, Q, K)).astype(np.float32)
    xbits = G._layout(G._bf16_bits(pkg, x), rows, pitch)
    y = pkg.bf16_bits_to_f32(G._fwd_run(eng, pkg, xbits, f, None, (N, H, W, C, K, R, S), stride=st, pitch=pitch, rows=rows))
    assert np.array_equal(y, CR.conv_fwd_f64(x, f, None, st))                  # exact: |y| <= 3 * R * S * C
    dyd = eng.to_device(G._bf16_bits(pkg, dy))
    dw = eng.array((K, R, S, C))
    eng.conv_wgrad(eng.to_device(xbits), dyd, dw, N, H, W, C, K, R, S, row_pitch=pitch, image_rows=rows, stride=st)
    dx = pkg.bf16_bits_to_f32(_dgrad(eng, dyd, f, N, H, W, C, K, R, S, st, pitch, rows))
    assert np.array_equal(dx, CS.conv_dgrad_f64(dy, f, H, W, st))            # exact in bf16 at these magnitudes
    a = float(np.sum(y.astype(np.float64) * dy))
    b = float(np.sum(x.astype(np.float64) * dx))
    c = float(np.sum(f.astype(np.float64) * dw.to_host()))
    assert a == b == c, (a, b, c)


SMALL = [  # N, H, W, C, K, R, S, stride
    (2, 40, 36, 3, 64, 3, 3, 2), (3, 28, 28, 1, 6, 5, 5, 2), (2, 23, 30, 2, 64, 3, 3, 3), (2, 25, 34, 1, 128, 3, 3, 4),
    (2, 30, 44, 1, 64, 7, 7, 2),
]


@pytest.mark.parametrize("case", SMALL, ids=["x".join(map(str, c)) for c in SMALL])
def test_strided_tensor_core_path_against_the_fma_path(eng, pkg, case):
    """The wgmma kernels against the FMA-pipe reference kernels at the same stride: weight gradient rel-L2 <= 1e-5, input
    gradients both within 2^-8 |ref| + 1e-3 of the float64 reference; tensor-core reruns bit-identical."""
    N, H, W, C, K, R, S, st = case
    P, Q = CS.out_size(H, W, R, S, st)
    rng = np.random.default_rng(sum(case))
    xb = G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C))
    dyb = G._uniform_bits(pkg, rng, -1, 1, (N, P, Q, K))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    pitch = (W * C + 7) // 8 * 8
    xd, dyd = eng.to_device(G._layout(xb, H, pitch)), eng.to_device(dyb)
    ref_dx = CS.conv_dgrad_f64(pkg.bf16_bits_to_f32(dyb), f, H, W, st)
    out = {}
    try:
        for path in ("tc", "fma"):
            eng.conv_bwd_select(reference=path == "fma")
            runs = []
            for _ in range(2):
                dw = eng.array((K, R, S, C))
                eng.conv_wgrad(xd, dyd, dw, N, H, W, C, K, R, S, row_pitch=pitch, stride=st)
                dx = pkg.bf16_bits_to_f32(_dgrad(eng, dyd, f, N, H, W, C, K, R, S, st, pitch, 0))
                runs.append((dw.to_host(), dx))
            out[path] = runs
    finally:
        eng.conv_bwd_select(reference=False)
    (tw, tx), (tw2, tx2) = out["tc"]
    assert np.array_equal(tw.view(np.uint32), tw2.view(np.uint32)) and np.array_equal(tx.view(np.uint32), tx2.view(np.uint32))
    fw = out["fma"][0][0].astype(np.float64)
    rel = np.linalg.norm(tw - fw) / np.linalg.norm(fw)
    assert rel <= 1e-5, rel
    for dx in (tx, out["fma"][0][1]):
        err = np.abs(dx - ref_dx)
        assert np.all(err <= 2.0 ** -8 * np.abs(ref_dx) + 1e-3), float(err.max())


WGRAD_PAD_STRIDED = [  # N, H, W, C, K, R, S, stride, row_pitch, image_rows
    (3, 151, 542, 1, 64, 3, 3, 2, 552, 160),            # guard (W*C*2 % 16 != 0), several pixel chunks
    (1024, 28, 28, 1, 6, 5, 5, 2, 32, 32),              # guard, LeNet c1 at pitch 32
    (7, 337, 136, 2, 64, 3, 3, 2, 288, 340),            # no guard, pitch > W*C
    (4, 4006, 40, 1, 64, 3, 3, 2, 48, 4010),            # ragged last row block, pad columns and rows
]


@pytest.mark.parametrize("case", WGRAD_PAD_STRIDED, ids=["x".join(map(str, c[:8])) + f"-p{c[8]}" for c in WGRAD_PAD_STRIDED])
def test_strided_weight_gradient_ignores_row_padding(eng, pkg, case):
    """NaN in the pad columns and rows of x: the strided weight gradient is bit-identical to the zero-padded run."""
    N, H, W, C, K, R, S, st, pitch, rows = case
    assert CS.wgrad_regime(pkg, N, H, W, C, K, R, S, G._sm(eng), st) is not None
    rng = np.random.default_rng(sum(case))
    P, Q = CS.out_size(H, W, R, S, st)
    xb = G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C))
    dyd = eng.to_device(G._uniform_bits(pkg, rng, -1, 1, (N, P, Q, K)))
    out = []
    for canvas in (G._layout(xb, rows, pitch), G._nan_padded(xb, rows, pitch)):
        dw = eng.array((K, R, S, C))
        eng.conv_wgrad(eng.to_device(canvas), dyd, dw, N, H, W, C, K, R, S, row_pitch=pitch, image_rows=rows, stride=st)
        out.append(dw.to_host())
    assert np.isfinite(out[0]).all()
    assert np.array_equal(out[1].view(np.uint32), out[0].view(np.uint32)), int(np.isnan(out[1]).sum())


@pytest.mark.parametrize("case", [CR.BWD_MULTI[i] for i in (1, 2, 5, 11)], ids=["lenet_c1", "k96", "c2_ragged", "c1_guard"])
def test_stride_1_through_the_strided_entry_points_is_bit_identical(eng, pkg, case):
    """pcnn_conv_wgrad_strided / pcnn_conv_dgrad_strided at stride 1 against pcnn_conv_wgrad / pcnn_conv_dgrad, both paths"""
    N, H, W, C, K, R, S, pitch, rows = case
    _p = importlib.import_module(type(eng).__module__)._p
    pitch_, rows_ = pitch or W * C, rows or H
    rng = np.random.default_rng(sum(case))
    xd = eng.to_device(G._layout(G._uniform_bits(pkg, rng, 0, 1, (N, H, W, C)), rows_, pitch_))
    dyd = eng.to_device(G._uniform_bits(pkg, rng, -1, 1, (N, H - R + 1, W - S + 1, K)))
    fd = eng.to_device(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32))
    try:
        for ref in (False, True):
            eng.conv_bwd_select(reference=ref)
            res = []
            for strided in (False, True):
                dw = eng.array((K, R, S, C))
                dx = eng.to_device(np.full((N, rows_, pitch_), NAN_BF16, np.uint16))
                tail = (1, int(pitch), int(rows)) if strided else (int(pitch), int(rows))
                sfx = "_strided" if strided else ""
                eng._call("pcnn_conv_wgrad" + sfx, _p(xd), _p(dyd), _p(dw), N, H, W, C, K, R, S, *tail)
                eng._call("pcnn_conv_dgrad" + sfx, _p(dyd), _p(fd), _p(dx), N, H, W, C, K, R, S, *tail)
                res.append((dw.to_host(), dx.to_host()))
            assert np.array_equal(res[0][0].view(np.uint32), res[1][0].view(np.uint32)), ref
            assert np.array_equal(res[0][1], res[1][1]), ref
    finally:
        eng.conv_bwd_select(reference=False)
