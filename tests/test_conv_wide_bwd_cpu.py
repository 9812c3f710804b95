"""Host-side checks of the wide-channel gradients (no GPU): pcnn_conv_wide_bwd_info has exactly the forward plan's domain and
refusals, reports the tiling of the benchmark layers, and puts every multi-tile GPU case in its regime."""
import pytest

import test_conv_wide_bwd_gpu as WB
import test_conv_wide_cpu as WC


def _accepts(fn, *a):
    try:
        fn(*a)
        return True
    except Exception as e:                                   # PcnnError
        assert getattr(e, "code", None) == -1, e
        return False


def test_backward_domain_is_the_wide_forward_domain(pkg):
    """Over the grid of test_every_shape_has_at_most_one_forward_kernel the backward query accepts exactly the shapes the wide
    forward query accepts."""
    N, H, W = 2, 20, 21
    accepted = 0
    for C in range(1, 73):
        for R in range(1, 8):
            for S in range(1, 8):
                for K in (6, 8, 64, 200, 256, 264):
                    for st in range(1, 5):
                        fwd = _accepts(pkg.conv_wide_plan_info, N, H, W, C, K, R, S, st)
                        assert _accepts(pkg.conv_wide_bwd_info, N, H, W, C, K, R, S, st) == fwd, (C, K, R, S, st)
                        accepted += fwd
    assert accepted > 5000


_REFUSALS = next(m for m in WC.test_wide_plan_refusals_name_their_rule.pytestmark if m.name == "parametrize").args[1]


@pytest.mark.parametrize("bad, msg", _REFUSALS)
def test_backward_refusals_name_their_rule(pkg, bad, msg):
    """Each refusal of the wide forward plan, with the same rule text, naming the backward query."""
    a = dict(N=2, H=28, W=28, C=64, K=64, R=3, S=3, stride=1, row_pitch=None, image_rows=0)
    a.update(bad)
    with pytest.raises(pkg.PcnnError, match=msg) as e:
        pkg.conv_wide_bwd_info(**a)
    assert e.value.code == -1
    assert "pcnn_conv_wide_bwd_info" in e.value.msg and "pcnn_conv_wide_plan_create" not in e.value.msg


def test_backward_query_reports_the_tiling_of_the_benchmark_layers(pkg):
    """The five layers of `conv_bench.py widebwd` at N = 128: weight-gradient row blocks, ranges of 32 pixel blocks of the
    forward's tiling, stages; input-gradient pixel block of the phase grid, groups, stages, tiles."""
    def q(*a, **k):
        b = pkg.conv_wide_bwd_info(*a, **k)
        return tuple(b[x] for x in ("wgrad_row_blocks", "wgrad_splits", "wgrad_blocks_per_split", "wgrad_stages", "wgrad_units",
                                    "dgrad_Pt", "dgrad_Qt", "dgrad_groups", "dgrad_stages", "dgrad_tiles"))
    assert q(128, 56, 56, 64, 64, 3, 3) == (9, 108, 32, 4, 540, 2, 64, 1, 8, 3584)
    assert q(128, 28, 28, 128, 128, 3, 3) == (18, 28, 32, 3, 252, 4, 32, 1, 5, 896)
    assert q(128, 14, 14, 256, 256, 3, 3) == (36, 8, 32, 2, 144, 8, 16, 1, 3, 256)
    assert q(128, 56, 56, 64, 256, 1, 1) == (1, 112, 32, 2, 112, 2, 64, 1, 8, 3584)
    # stride 2: four phases of 28 x 28 pixels, each 7 blocks of 4 x 32 per image
    assert q(128, 56, 56, 64, 128, 3, 3, 2) == (9, 28, 32, 3, 140, 4, 32, 1, 8, 4 * 7 * 128)
    # C = 320: two channel groups; the phases of stride 4 on 19 x 18 pixels; tiny shapes have one range
    assert pkg.conv_wide_bwd_info(2, 12, 13, 320, 64, 3, 3)["dgrad_groups"] == 2
    assert pkg.conv_wide_bwd_info(2, 12, 13, 320, 64, 3, 3)["wgrad_row_blocks"] == 9 * 5
    assert pkg.conv_wide_bwd_info(2, 19, 18, 40, 24, 2, 3, 4)["dgrad_tiles"] == 2 * 16
    assert pkg.conv_wide_bwd_info(3, 14, 14, 16, 8, 3, 3)["wgrad_splits"] == 1
    # a pitch and an image pitch change nothing in the tiling
    assert pkg.conv_wide_bwd_info(4, 31, 29, 40, 120, 3, 3, 2, 29 * 40 + 8, 33) == pkg.conv_wide_bwd_info(4, 31, 29, 40, 120, 3, 3, 2)


@pytest.mark.parametrize("sm_count", [114, 132])
def test_wide_backward_multi_tile_cases_reach_their_regime(pkg, sm_count):
    """Weight gradient: more than 2 x stages pixel blocks per work unit and more work units than SMs.  Input gradient: more than
    2 x stages tiles on every CTA."""
    for case in WB.MULTI:
        w, d = WB.regime(pkg, case[:8], sm_count)
        assert w["blocks_per_unit"] > 2 * w["stages"] and w["units"] > sm_count, (case, w)
        assert d["min_tiles_per_cta"] > 2 * d["stages"], (case, d)
