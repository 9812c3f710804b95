"""Host-side checks of zero padding for the wide-channel convolution (no GPU): the padded float64 references equal PyTorch's
conv2d and its gradients, the _padded queries at padding (0, 0) are the unpadded ones, the padded domain rule, the new refusals
and their messages, and the regime the padded multi-tile GPU cases reach."""
import ctypes

import numpy as np
import pytest
import torch

import test_conv_wide_pad_gpu as PG


@pytest.mark.parametrize("case", PG.CASES, ids=PG.ids(PG.CASES))
def test_padded_references_are_torch_conv2d(case):
    """np.pad + conv_ref / conv_ref_strided (dx cropped) against torch.nn.functional.conv2d, torch.nn.grad.conv2d_weight and
    conv2d_input in float64 with the same (stride, padding), at N = 1."""
    _, H, W, C, K, R, S, st, ph, pw = case[:10]
    C, K = min(C, 24), min(K, 16)                            # the formulas do not depend on the channel counts
    rng = np.random.default_rng(sum(case))
    P, Q = PG.out_size(H, W, R, S, st, ph, pw)
    x = rng.standard_normal((1, H, W, C))
    f = rng.standard_normal((K, R, S, C))
    b = rng.standard_normal(K)
    dy = rng.standard_normal((1, P, Q, K))
    xt, ft, dyt = (torch.from_numpy(a).permute(0, 3, 1, 2) for a in (x, f, dy))
    y = torch.nn.functional.conv2d(xt, ft, torch.from_numpy(b), stride=st, padding=(ph, pw)).permute(0, 2, 3, 1).numpy()
    np.testing.assert_allclose(PG.fwd_ref(x, f, b, st, ph, pw), y, rtol=1e-12, atol=1e-12)
    dw = torch.nn.grad.conv2d_weight(xt, ft.shape, dyt, stride=st, padding=(ph, pw)).permute(0, 2, 3, 1).numpy()
    np.testing.assert_allclose(PG.wgrad_ref(x, dy, R, S, st, ph, pw), dw, rtol=1e-12, atol=1e-12)
    dx = torch.nn.grad.conv2d_input(xt.shape, ft, dyt, stride=st, padding=(ph, pw)).permute(0, 2, 3, 1).numpy()
    np.testing.assert_allclose(PG.dgrad_ref(dy, f, H, W, st, ph, pw), dx, rtol=1e-12, atol=1e-12)


def _raw(pkg, name, nout, *args):
    """(status, outputs or the error text) of a host-only query called through its C symbol"""
    out = (ctypes.c_int * nout)()
    rc = getattr(pkg.lib(), name)(*args, out)
    return (rc, tuple(out)) if rc == 0 else (rc, pkg.lib().pcnn_last_error_string().decode())


def test_padded_queries_at_zero_padding_are_the_unpadded_ones(pkg):
    """Over the grid of test_every_shape_has_at_most_one_forward_kernel: at padding (0, 0) the two _padded queries accept,
    refuse and report exactly what the unpadded ones do, with the same rule text naming the padded call."""
    N, H, W = 2, 20, 21
    accepted = 0
    for C in range(1, 73):
        pitch = (W * C + 7) // 8 * 8
        for R in range(1, 8):
            for S in range(1, 8):
                for K in (6, 8, 64, 200, 256, 264):
                    for st in range(1, 5):
                        a = (N, H, W, C, K, R, S, st)
                        for base, padded, create, nout in (
                                ("pcnn_conv_wide_plan_info", "pcnn_conv_wide_plan_info_padded", "pcnn_conv_wide_plan_create", 8),
                                ("pcnn_conv_wide_bwd_info", "pcnn_conv_wide_bwd_info_padded", "pcnn_conv_wide_bwd_info", 10)):
                            rc0, v0 = _raw(pkg, base, nout, *a, pitch, 0)
                            rc1, v1 = _raw(pkg, padded, nout, *a, 0, 0, pitch, 0)
                            assert rc1 == rc0, (a, base, v0, v1)
                            if rc0 == 0:
                                assert v1 == v0, (a, base)
                            else:
                                assert v1 == v0.replace(create + ":", create + "_padded:"), (a, v0, v1)
                        accepted += rc0 == 0
    assert accepted > 5000


def _rule(pkg, N, H, W, C, K, R, S, st, ph, pw):
    """the padded domain of include/pcnn.h, restated"""
    if not (1 <= st <= 4 and 1 <= R <= 7 and 1 <= S <= 7 and 0 <= ph <= R - 1 and 0 <= pw <= S - 1):
        return False
    if not (N > 0 and H + 2 * ph >= R and W + 2 * pw >= S and C > 0 and K > 0):
        return False
    if (ph > 0 and H < st) or (pw > 0 and W < st):
        return False
    if not (C % 8 == 0 and K % 8 == 0 and K <= 256):
        return False
    if (ph, pw) == (0, 0):
        try:
            pkg.conv_tc_plan_info(N, H, W, C, K, R, S, st)
            return False
        except pkg.PcnnError:
            pass
    return True


def _accepts(fn, *a, **k):
    try:
        fn(*a, **k)
        return True
    except Exception as e:                                   # PcnnError
        assert getattr(e, "code", None) == -1, e
        return False


def test_padded_domain_is_the_rule(pkg):
    """Over R, S in 1..7, stride 1..4, every pad from 0 to R (S), small H and W (H < R, H < stride and H = stride among them) and
    a few C / K: both padded queries accept exactly the shapes of the domain rule, and the forward and backward agree."""
    accepted = refused = 0
    for C, K in ((64, 32), (8, 8), (40, 264), (36, 64)):
        for R in range(1, 8):
            for S in range(1, 8):
                for st in range(1, 5):
                    for ph in range(0, R + 1):
                        for pw in range(0, S + 1):
                            for H, W in ((1, 3), (2, 2), (3, 9), (4, 1), (5, 4), (9, 6)):
                                want = _rule(pkg, 2, H, W, C, K, R, S, st, ph, pw)
                                a = (2, H, W, C, K, R, S, st)
                                assert _accepts(pkg.conv_wide_plan_info, *a, padding=(ph, pw)) == want, (a, ph, pw)
                                assert _accepts(pkg.conv_wide_bwd_info, *a, padding=(ph, pw)) == want, (a, ph, pw)
                                accepted += want
                                refused += not want
    assert accepted > 5000 and refused > 5000, (accepted, refused)


def test_padding_lets_the_wide_plan_take_row_toeplitz_shapes(pkg):
    """C = K = 8 with 3x3 taps: the row-Toeplitz plan's shape unpadded, the wide plan's padded (it alone pads)."""
    pkg.conv_tc_plan_info(2, 8, 8, 8, 8, 3, 3)
    with pytest.raises(pkg.PcnnError, match="pcnn_conv_tc_plan_create"):
        pkg.conv_wide_plan_info(2, 8, 8, 8, 8, 3, 3)
    assert pkg.conv_wide_plan_info(2, 8, 8, 8, 8, 3, 3, padding=(1, 1))["useful_pixels"] == 2 * 8 * 8
    assert pkg.conv_wide_plan_info(2, 8, 8, 8, 8, 3, 3, padding=(0, 1))["useful_pixels"] == 2 * 6 * 8


@pytest.mark.parametrize("bad, msg", [
    (dict(padding=(3, 1)), r"padding \(3, 1\) with R = 3, S = 3 taps: 0 <= pad_h <= R - 1"),
    (dict(padding=(1, -1)), r"padding \(1, -1\) with R = 3, S = 3 taps: .*0 <= pad_w <= S - 1"),
    (dict(H=1, padding=(0, 1)), r"bad shape N=2 H=1 .* padding \(0, 1\): H \+ 2\*pad_h >= R"),
    (dict(W=0, padding=(1, 1)), r"bad shape N=2 H=28 W=0 .* padding \(1, 1\): .*W \+ 2\*pad_w >= S"),
    (dict(H=3, stride=4, padding=(1, 1)), r"H = 3, W = 28 with padding \(1, 1\) at stride 4: a padded direction needs at least "
                                          r"stride rows / pixels, so that every phase of x has one inside the image"),
    (dict(W=2, R=1, stride=3, padding=(0, 1)), r"H = 28, W = 2 with padding \(0, 1\) at stride 3"),
    (dict(C=36, padding=(1, 1)), r"C % 8"),                 # the unpadded rules hold with padding, naming the padded call
    (dict(K=264, padding=(1, 1)), r"K <= 256"),
    (dict(stride=5, padding=(1, 1)), "stride 5 outside 1..4"),
    (dict(image_rows=27, padding=(1, 1)), "smaller than H"),
])
def test_padded_refusals_name_their_rule_and_the_call(pkg, bad, msg):
    a = dict(N=2, H=28, W=28, C=64, K=64, R=3, S=3, stride=1, row_pitch=None, image_rows=0)
    a.update(bad)
    for fn, name in ((pkg.conv_wide_plan_info, "pcnn_conv_wide_plan_create_padded"),
                     (pkg.conv_wide_bwd_info, "pcnn_conv_wide_bwd_info_padded")):
        with pytest.raises(pkg.PcnnError, match=msg) as e:
            fn(**a)
        assert e.value.code == -1                            # PCNN_ERR_ARG
        assert e.value.msg.startswith(name + ":"), e.value.msg


def test_padded_queries_report_the_padded_sizes(pkg):
    """The four `conv_bench.py widesame` layers at N = 128: P x Q output pixels of the padded image, and the tiling of the valid
    convolution on the canvas (the same tiles)."""
    for H, W, C, K, st in ((56, 56, 64, 64, 1), (28, 28, 128, 128, 1), (14, 14, 256, 256, 1), (56, 56, 64, 128, 2)):
        pl = pkg.conv_wide_plan_info(128, H, W, C, K, 3, 3, st, padding=(1, 1))
        P, Q = PG.out_size(H, W, 3, 3, st, 1, 1)
        assert pl["useful_pixels"] == 128 * P * Q and (P, Q) == (H // st, W // st)
        canvas = pkg.conv_wide_plan_info(128, H + 2, W + 2, C, K, 3, 3, st)
        assert pl == canvas
        b = pkg.conv_wide_bwd_info(128, H, W, C, K, 3, 3, st, padding=(1, 1))
        assert {k: v for k, v in b.items() if k.startswith("wgrad")} == \
            {k: v for k, v in pkg.conv_wide_bwd_info(128, H + 2, W + 2, C, K, 3, 3, st).items() if k.startswith("wgrad")}
        # the input gradient tiles the phases of dx (H x W), not those of the canvas
        assert b["dgrad_tiles"] == pkg.conv_wide_bwd_info(128, H, W, C, K, 3, 3, st)["dgrad_tiles"]


@pytest.mark.parametrize("sm_count", [114, 132])
def test_padded_multi_tile_cases_reach_their_regime(pkg, sm_count):
    """Forward: more than 2 x stages tiles on every CTA.  Weight gradient: more than 2 x stages pixel blocks per work unit and
    more work units than SMs.  Input gradient: more than 2 x stages tiles on every CTA."""
    for case in PG.MULTI:
        g = PG.regime(pkg, case, sm_count)
        assert PG.in_regime(g, sm_count), (case, g)
