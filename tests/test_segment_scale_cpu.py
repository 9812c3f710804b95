"""Host-only checks behind test_segment_scale_gpu.py: every shape it runs has the tiling, grid and laps it is there for (pinned at an
H100 SXM's 132 SMs), and its float64 reference of the transposed convolution, torch's CPU conv_transpose2d and autograd, equals
segment_ref's on the small shapes of test_segment_gpu.py."""
import numpy as np
import pytest

import segment_ref as SR
import test_segment_gpu as SG
import test_segment_scale_gpu as SS

SM = 132


def test_convt_scale_shapes_tiling(pkg):
    got = [SS.coverage(pkg, s) for s in SS.CONVT_SCALE]
    assert [(c["tiles"], c["groups"], c["wgrad_splits"], c["wgrad_max_blocks"]) for c in got] == [
        (512, 1, 4, 32), (1024, 1, 8, 32), (3584, 1, 28, 32), (512, 1, 4, 32), (576, 1, 2, 32), (128, 2, 2, 32)]
    for s in SS.CONVT_SCALE:
        SS.assert_coverage(pkg, s, SM)


def test_convt_scale_shapes_reach_their_paths(pkg):
    """C_out 24 pads the MMA columns; the stride-3 shape has phases without a tap; the last shape has two groups of 256 and 8"""
    N, H, W, Ci, Co, R, S, st, pad, op = SS.CONVT_SCALE[3]
    assert Co % 16 != 0
    N, H, W, Ci, Co, R, S, st, pad, op = SS.CONVT_SCALE[4]
    taps_h = [len(range((a + pad[0]) % st, R, st)) for a in range(st)]
    taps_w = [len(range((b + pad[1]) % st, S, st)) for b in range(st)]
    assert R < st and S < st and 0 in taps_h and 0 in taps_w and max(taps_h) > 0
    assert SS.CONVT_SCALE[5][4] > 256


def test_convt_pitched_shapes_tiling(pkg):
    (s0, p0, r0), (s1, p1, r1) = SS.PITCHED
    i = pkg.conv_transpose_info(*s0[:10], row_pitch=p0, image_rows=r0)
    assert (i["H_out"], i["W_out"], i["row_pitch"], i["image_rows"]) == (28, 28, 1800, 30) and p0 > 28 * 64
    assert SS.coverage(pkg, s0, p0, r0) == dict(tiles=1024, groups=1, wgrad_splits=8, wgrad_max_blocks=32)
    i = pkg.conv_transpose_info(*s1[:10], row_pitch=p1, image_rows=r1)
    assert (i["H_out"], i["W_out"], i["row_pitch"], i["image_rows"]) == (10, 12, 328, 12) and p1 > 12 * 24


def test_pixel_ce_shapes_take_laps():
    """both kernels of the pixel loss run at least two laps at every pixel count, the benchmark's about 6 and 95"""
    for _, P, _ in SS.PIXEL_CE:
        assert P > 4 * SM * 256 and SS.count_laps(P, SM) >= 2 and SS.ce_laps(P, SM) >= 2
    assert (SS.count_laps(16 * 224 * 224, SM), SS.ce_laps(16 * 224 * 224, SM)) == (6, 96)
    assert (SS.count_laps(150_000, SM), SS.ce_laps(150_000, SM)) == (2, 18)


def test_upsample_shapes_grid(pkg):
    for N, H, W, C, f in SS.UPSAMPLE_BENCH:
        i = pkg.upsample_bilinear_info(N, H, W, C, H * f, W * f)
        assert i["grid_fwd"] < SS.UP_GRID_CAP and i["vec"] == (8 if C % 8 == 0 else 1)
    fwd, bwd = (pkg.upsample_bilinear_info(*c[:6]) for c in SS.UPSAMPLE_CAP)
    assert (fwd["grid_fwd"], fwd["vec"], bwd["grid_bwd"], bwd["vec"]) == (1 << 20, 1, 1 << 20, 1)
    for N, H, W, C, Ho, Wo, pas in SS.UPSAMPLE_CAP:        # 285 M items; the last image starts on the second lap
        items = N * C * (Ho * Wo if pas == "fwd" else H * W)
        assert items == 285_212_672 and items * (N - 1) // N == SS.UP_GRID_CAP * 256


@pytest.mark.parametrize("shape", SG.CONVT)
@pytest.mark.parametrize("operands", ["integer", "random"])
def test_torch_convt_reference_is_segment_ref(shape, operands):
    """the forward and both gradients: exactly equal on integer operands (both sums are exact in float64), within 1e-12 on random"""
    N, H, W, Ci, Co, R, S, st, pad, op = shape
    rng = np.random.default_rng(sum(shape[:8]))
    draw = (lambda shp: SG.ints(rng, shp).astype(np.float64)) if operands == "integer" else rng.standard_normal
    x, w, b = draw((N, H, W, Ci)), draw((Ci, Co, R, S)), draw(Co)
    pre, _ = SR.convt_fwd_f64(x, w, b, st, pad, op)
    dy = draw(pre.shape)
    rdx, rdw, _ = SR.convt_bwd_f64(x, w, dy, st, pad)
    for got, want in zip(SS.torch_convt(shape, x, w, b, dy), (pre, rdx, rdw)):
        if operands == "integer":
            assert np.array_equal(got, want)
        else:
            np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
