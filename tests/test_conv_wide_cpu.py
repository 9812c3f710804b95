"""Host-side checks of the wide-channel forward plan (no GPU): the partition of shapes between the row-Toeplitz plan and the wide
plan, each refusal and its message, and the regime the multi-tile GPU cases reach."""
import pytest

import test_conv_wide_gpu as WG


def test_every_shape_has_at_most_one_forward_kernel(pkg):
    """Over C in 1..72, R and S in 1..7, K in {6, 8, 64, 200, 256, 264}, stride 1..4: the two plan queries never both accept, and
    the wide plan accepts exactly the shapes of its domain rule."""
    N, H, W = 2, 20, 21
    accepted = 0
    for C in range(1, 73):
        for R in range(1, 8):
            for S in range(1, 8):
                for K in (6, 8, 64, 200, 256, 264):
                    for st in range(1, 5):
                        try:
                            pkg.conv_tc_plan_info(N, H, W, C, K, R, S, st)
                            tc = True
                        except pkg.PcnnError:
                            tc = False
                        try:
                            pkg.conv_wide_plan_info(N, H, W, C, K, R, S, st)
                            wide = True
                        except pkg.PcnnError:
                            wide = False
                        assert not (tc and wide), (C, K, R, S, st)
                        assert wide == (not tc and C % 8 == 0 and K % 8 == 0 and K <= 256), (C, K, R, S, st)
                        accepted += wide
    assert accepted > 5000


@pytest.mark.parametrize("bad, msg", [
    (dict(C=8, S=3), "pcnn_conv_tc_plan_create"),            # (Qt-1+3)*8 <= 32 at Qt = 2: the row-Toeplitz plan takes it
    (dict(C=16, R=1, S=1), "pcnn_conv_tc_plan_create"),      # 1x1, S*C = 16
    (dict(C=36), r"C % 8"),
    (dict(C=60), r"C % 8"),
    (dict(K=60), r"K % 8"),
    (dict(K=264), r"K <= 256"),
    (dict(R=8), "taps must be 1..7"),
    (dict(S=9), "taps must be 1..7"),
    (dict(stride=0), "stride 0 outside 1..4"),
    (dict(stride=5), "stride 5 outside 1..4"),
    (dict(row_pitch=28 * 64 + 4), "multiple of 8"),
    (dict(row_pitch=28 * 64 - 8), ">= W\\*C"),
    (dict(image_rows=27), "smaller than H"),
])
def test_wide_plan_refusals_name_their_rule(pkg, bad, msg):
    a = dict(N=2, H=28, W=28, C=64, K=64, R=3, S=3, stride=1, row_pitch=None, image_rows=0)
    a.update(bad)
    with pytest.raises(pkg.PcnnError, match=msg) as e:
        pkg.conv_wide_plan_info(**a)
    assert e.value.code == -1                                # PCNN_ERR_ARG
    assert "pcnn_conv_wide_plan_create" in e.value.msg


def test_wide_plan_query_reports_tiling_and_waste(pkg):
    """The tiling of the benchmark layers: pixel blocks, chunks, stages, tiles, and the output pixels they issue."""
    small = pkg.conv_wide_plan_info(128, 14, 14, 256, 256, 3, 3)       # 12x12 outputs
    assert (small["Pt"], small["Qt"], small["chunks"], small["npad"]) == (8, 16, 4, 256)
    assert small["tiles"] == 128 * 2 and small["issued_pixels"] == 128 * 256 and small["useful_pixels"] == 128 * 144
    big = pkg.conv_wide_plan_info(128, 56, 56, 64, 64, 3, 3)           # 54x54 outputs: 27 blocks of 2 x 64
    assert (big["Pt"], big["Qt"], big["n_pb"], big["n_qb"], big["chunks"]) == (2, 64, 27, 1, 1)
    assert big["issued_pixels"] == 128 * 27 * 128 and big["stages"] == 8
    s2 = pkg.conv_wide_plan_info(128, 56, 56, 64, 128, 3, 3, stride=2)  # 27x27 outputs
    assert s2["useful_pixels"] == 128 * 27 * 27 and s2["issued_pixels"] == s2["tiles"] * 128
    # rows per image need not be a multiple of the stride, and a pitch / image pitch changes nothing in the tiling
    assert pkg.conv_wide_plan_info(4, 31, 29, 40, 120, 3, 3, 2, 29 * 40 + 8, 33)["tiles"] == \
        pkg.conv_wide_plan_info(4, 31, 29, 40, 120, 3, 3, 2)["tiles"]
    for shape in WG.WIDE_CASES + WG.WIDE_MULTI:
        pl = pkg.conv_wide_plan_info(*shape)
        assert pl["Pt"] * pl["Qt"] == 128 and pl["issued_pixels"] >= pl["useful_pixels"]
        assert 2 <= pl["stages"] <= 8


@pytest.mark.parametrize("sm_count", [114, 132])
def test_wide_multi_tile_cases_reach_their_regime(pkg, sm_count):
    """Every multi-tile GPU case runs more than 2 x stages tiles on every CTA of a 114- and a 132-SM part."""
    for N, H, W, C, K, R, S, st in WG.WIDE_MULTI:
        g = WG.wide_regime(pkg, N, H, W, C, K, R, S, st, sm_count)
        assert g["min_tiles_per_cta"] > 2 * g["stages"], ((N, H, W, C, K, R, S, st), g)
