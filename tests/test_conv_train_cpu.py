"""Host-side parts of training a convolution layer (no GPU): the family ConvLayer picks for a shape agrees with the two plans'
queries, and the numpy float32 replay of the sigmoid derivative that the GPU tests compare pcnn_conv_bias_act_bwd against agrees
with a float64 evaluation within bf16 rounding."""
import itertools

import numpy as np
import pytest


def _accepts(fn, *args, **kw):
    try:
        fn(*args, **kw)
        return True
    except Exception as e:                      # the queries raise PcnnError
        if type(e).__name__ != "PcnnError":
            raise
        return False


SHAPES = list(itertools.product([2], [9, 28], [11, 28], [1, 3, 8, 64], [6, 8, 16, 64], [1, 3, 5], [3, 5], [1, 2],
                                [(0, 0), (1, 1), (0, 2)]))


def test_family_agrees_with_plan_queries(pkg):
    counts = {"narrow": 0, "wide": 0, "refused": 0, "refused_pad_copy": 0}
    for N, H, W, C, K, R, S, st, (ph, pw) in SHAPES:
        if ph >= R or pw >= S:
            continue
        tc = _accepts(pkg.conv_tc_plan_info, N, H, W, C, K, R, S, st)
        wide = _accepts(pkg.conv_wide_plan_info, N, H, W, C, K, R, S, st, padding=(ph, pw))
        try:
            fam = pkg.conv_layer_family(N, H, W, C, K, R, S, st, padding=(ph, pw))
        except pkg.PcnnError as e:
            fam = None
            msg = str(e)
        if (ph, pw) == (0, 0):
            assert not (tc and wide), "the two forward plans overlap"
            want = "narrow" if tc else ("wide" if wide else None)
        else:
            want = "wide" if wide else None
        assert fam == want, (N, H, W, C, K, R, S, st, ph, pw, fam)
        if fam is None:
            pad_copy = (ph, pw) != (0, 0) and tc
            assert ("pcnn_pad_nhwc_bf16" in msg) == pad_copy, msg
            counts["refused_pad_copy" if pad_copy else "refused"] += 1
        else:
            counts[fam] += 1
    assert all(v > 0 for v in counts.values()), counts


def test_narrow_padded_shape_is_refused(pkg):
    with pytest.raises(pkg.PcnnError, match="pcnn_pad_nhwc_bf16"):
        pkg.conv_layer_family(64, 28, 28, 1, 6, 5, 5, padding=(2, 2))
    assert pkg.conv_layer_family(64, 28, 28, 1, 6, 5, 5) == "narrow"
    assert pkg.conv_layer_family(2, 8, 8, 8, 8, 3, 3) == "narrow"
    assert pkg.conv_layer_family(2, 8, 8, 8, 8, 3, 3, padding=(1, 1)) == "wide"       # padded: the wide plan's alone


def test_sigmoid_derivative_replay_within_bf16_rounding(pkg):
    """dpre = bf16(dy * (y * (1 - y))) in float32 against dy * y * (1 - y) in float64 on the same bf16 operands: the three float32
    roundings add at most 3 * 2^-24 relative, the bf16 rounding (8 significant bits) 2^-8"""
    import test_conv_train_gpu as T
    rng = np.random.default_rng(0)
    y, dy = T.random_operands(pkg, rng, 20000, 16)
    got = pkg.bf16_bits_to_f32(T.dpre_replay(pkg, y, dy)).astype(np.float64)
    yf, gf = pkg.bf16_bits_to_f32(y).astype(np.float64), pkg.bf16_bits_to_f32(dy).astype(np.float64)
    ref = gf * yf * (1.0 - yf)
    assert np.all(np.abs(got - ref) <= (2.0 ** -8 + 4 * 2.0 ** -24) * np.abs(ref) + 1e-38)
    assert np.array_equal(T.dpre_replay(pkg, y, pkg.f32_to_bf16_bits(np.zeros_like(gf, np.float32))), np.zeros_like(y))
