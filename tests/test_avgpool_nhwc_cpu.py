"""Host-side parts of the NHWC average pools (no GPU): the replays of tests/avgpool_ref.py agree with torch's CPU float64
avg_pool2d (both count_include_pad values), adaptive_avg_pool2d(x, 1) and their autograd backward, on the window shapes of the
max pool's tests with +-0, +-Inf and NaN; pcnn_avgpool_nhwc_info accepts exactly the max pool's domain; pcnn_global_avgpool_nhwc_info
accepts exactly its stated domain, names each refused rule, and partitions a shape as a function of the shape alone."""
import itertools

import numpy as np
import pytest
import torch

import avgpool_ref as AR
import maxpool_ref as MR
from test_maxpool_nhwc_cpu import CASES, cover_brute, domain_refusal, special_input

F = torch.nn.functional


def same(a, b, exact):
    """equal values (NaN where NaN; -0 == +0: torch sums from +0, so a window of all -0 gives it +0 where the rule gives -0)"""
    if exact:
        return np.array_equal(a, b, equal_nan=True)
    return np.allclose(a, b, rtol=1e-13, atol=0, equal_nan=True)


@pytest.mark.parametrize("include_pad", [0, 1])
@pytest.mark.parametrize("case", CASES, ids=["x".join(map(str, c)) for c in CASES])
def test_windowed_reference_matches_torch_cpu(case, include_pad):
    N, H, W, C, R, S, st, ph, pw = case
    rng = np.random.default_rng(sum(case) + include_pad)
    P, Q = MR.out_size(H, W, R, S, st, ph, pw)
    for kind, x in (("special", special_input(rng, (N, H, W, C), np.float64)), ("integer", rng.integers(-4, 5, (N, H, W, C)).astype(np.float64)),
                    ("random", rng.standard_normal((N, H, W, C)))):
        xt = torch.from_numpy(x).permute(0, 3, 1, 2).requires_grad_(True)
        y = F.avg_pool2d(xt, (R, S), st, (ph, pw), count_include_pad=bool(include_pad))
        assert tuple(y.shape) == (N, C, P, Q)
        got = AR.fwd(x, R, S, st, ph, pw, include_pad)
        assert same(y.detach().permute(0, 2, 3, 1).numpy(), got, kind == "integer"), kind
        dy = rng.standard_normal((N, P, Q, C)) if kind == "random" else rng.integers(-3, 4, (N, P, Q, C)).astype(np.float64)
        y.backward(torch.from_numpy(dy).permute(0, 3, 1, 2))
        dx, terms = AR.bwd(dy, H, W, R, S, st, ph, pw, include_pad)
        assert same(xt.grad.permute(0, 2, 3, 1).numpy(), dx, False), kind
        assert np.all(dx[:, terms == 0] == 0) and not np.signbit(dx[:, terms == 0]).any()
        # the float32 replays stay within the float32 rounding of the float64 references
        x32, dy32 = x.astype(np.float32), dy.astype(np.float32)
        fin = np.isfinite(got)
        y32 = AR.fwd(x32, R, S, st, ph, pw, include_pad).astype(np.float64)
        assert np.array_equal(np.isnan(y32), np.isnan(got)) and np.all(np.abs(y32 - got)[fin] <= 2.0 ** -20 * (1 + np.abs(got[fin]) * 50))
        dx32 = AR.bwd(dy32, H, W, R, S, st, ph, pw, include_pad)[0].astype(np.float64)
        assert np.all(np.abs(dx32 - dx) <= 2.0 ** -20 * (1 + np.abs(dx) * 50))


def test_windowed_reference_special_windows():
    """-0 windows keep -0 (the sum starts from the first term), +Inf with -Inf is NaN, NaN propagates, one Inf stays Inf"""
    ninf, inf, nan = -np.inf, np.inf, np.nan
    rows = [[-0.0, -0.0, -0.0, -0.0], [inf, ninf, 1, 2], [nan, 1, 2, 3], [inf, 1, 2, 3], [1, 2, 4, 8]]
    x = np.array(rows, np.float32).reshape(len(rows), 1, 4, 1)
    y = AR.fwd(x, 1, 4, 1, 0, 0, 1)[:, 0, 0, 0]
    assert y[0] == 0 and np.signbit(y[0]) and np.isnan(y[1]) and np.isnan(y[2]) and y[3] == np.inf and y[4] == np.float32(15 / 4)
    yt = F.avg_pool2d(torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2), (1, 4))[:, 0, 0, 0].numpy()
    assert yt[0] == 0 and np.isnan(yt[1]) and np.isnan(yt[2]) and yt[3] == np.inf and yt[4] == 15 / 4
    # the division is IEEE: 1/3 of a sum, not the sum times a rounded 1/3
    v = np.float32(0.1)
    x3 = np.full((1, 1, 3, 1), v, np.float32)
    s = np.float32(np.float32(v + v) + v)
    assert AR.fwd(x3, 1, 3, 1, 0, 0, 1)[0, 0, 0, 0] == s / np.float32(3)


@pytest.mark.parametrize("shape", [(2, 1, 1, 3), (2, 7, 7, 6), (3, 5, 9, 8), (2, 56, 56, 16), (1, 16, 33, 300)])
def test_global_reference_matches_torch_cpu(pkg, shape):
    N, H, W, C = shape
    rng = np.random.default_rng(sum(shape))
    info = pkg.global_avgpool_nhwc_info(N, H, W, C)
    for kind, x in (("integer", rng.integers(-8, 9, shape).astype(np.float64)), ("random", rng.standard_normal(shape)),
                    ("special", special_input(rng, shape, np.float64))):
        xt = torch.from_numpy(x).permute(0, 3, 1, 2).requires_grad_(True)
        y = F.adaptive_avg_pool2d(xt, 1)
        ref = AR.global_f64(x)
        assert same(y.detach()[:, :, 0, 0].numpy(), ref, False), kind
        assert same(xt.mean((2, 3)).detach().numpy(), ref, False), kind
        dy = rng.standard_normal((N, C))
        y.backward(torch.from_numpy(dy)[:, :, None, None])
        assert same(xt.grad.permute(0, 2, 3, 1).numpy(), AR.global_bwd(dy, H, W), False)
        y32 = AR.global_fwd(x.astype(np.float32), info)
        assert np.array_equal(np.isnan(y32), np.isnan(ref))
        if kind == "integer":                                          # exact sums: any order gives the same bits
            assert np.array_equal(y32, x.sum(axis=(1, 2)).astype(np.float32) / np.float32(H * W))


# ------------------------------------------------------------------------------------------------ info queries
def test_avgpool_info_is_the_max_pool_domain(pkg):
    """the same accepted shapes, outputs and refusals as the max pool (one pool_shape), with the function's own name"""
    counts = {"accepted": 0, "refused": 0}
    for R, S, st in itertools.product(range(1, 8), range(1, 8), range(1, 8)):
        for ph, pw in itertools.product(range(R // 2 + 2), range(S // 2 + 2)):
            for H, W in ((1, 4), (3, 7), (11, 1), (6, 4)):
                C = 3 if (R + S + st) % 2 else 16
                rule = domain_refusal(1, H, W, C, R, S, st, ph, pw)
                try:
                    info = pkg.avgpool_nhwc_info(1, H, W, C, R, S, st, (ph, pw))
                except pkg.PcnnError as e:
                    assert rule is not None and rule in e.msg and "pcnn_avgpool_nhwc_info" in e.msg, (R, S, st, ph, pw, H, W, e.msg)
                    counts["refused"] += 1
                    continue
                assert rule is None, (R, S, st, ph, pw, H, W)
                counts["accepted"] += 1
                assert info == pkg.maxpool_nhwc_info(1, H, W, C, R, S, st, (ph, pw))
                P, Q = info["P"], info["Q"]
                assert info["cover"] == cover_brute(H, R, st, ph, P) * cover_brute(W, S, st, pw, Q)
                if (H + W + R) % 4 == 0:
                    for cip in (False, True):
                        y = F.avg_pool2d(torch.zeros(1, 1, H, W), (R, S), st, (ph, pw), count_include_pad=cip)
                        assert tuple(y.shape[2:]) == (P, Q)
                        if cip:                                      # torch's divisor is R*S wherever the rule says so
                            ones = F.avg_pool2d(torch.ones(1, 1, H, W, dtype=torch.float64), (R, S), st, (ph, pw), count_include_pad=True)
                            want = AR.counts(H, W, R, S, st, ph, pw, 0) / (R * S)
                            assert np.allclose(ones[0, 0].numpy(), want, rtol=1e-15)
    assert counts["accepted"] > 500 and counts["refused"] > 500, counts
    with pytest.raises(pkg.PcnnError, match="pcnn_avgpool_nhwc_info: image_rows 3: 0 \\(P\\) or >= P = 4"):
        pkg.avgpool_nhwc_info(1, 8, 8, 6, 2, 2, 2, image_rows=3)


def global_refusal(N, H, W, C, pitch):
    if min(N, H, W, C) < 1:
        return "each must be >= 1"
    if H * W * C > 2 ** 31 - 1 - 256:
        return "32-bit index range"
    if pitch != 0 and (pitch < C or pitch % 8):
        return f"row_pitch {pitch}: 0 (C rounded up to 8) or a multiple of 8 that is >= C = {C}"
    return None


def test_global_info_domain_and_partition(pkg):
    accepted = refused = 0
    for N, H, W, C, pitch in itertools.product((0, 1, 5), (0, 1, 7, 56), (1, 3, 56), (0, 1, 6, 8, 300, 2048, 4096), (0, 8, 300, 304, 2056)):
        rule = global_refusal(N, H, W, C, pitch)
        try:
            info = pkg.global_avgpool_nhwc_info(N, H, W, C, pitch)
        except pkg.PcnnError as e:
            assert rule is not None and rule in e.msg and "pcnn_global_avgpool_nhwc_info" in e.msg, (N, H, W, C, pitch, e.msg)
            refused += 1
            continue
        assert rule is None, (N, H, W, C, pitch)
        accepted += 1
        HW = H * W
        vec = 8 if C % 8 == 0 else 1
        G = C // vec
        assert info["row_pitch"] == (pitch or (C + 7) // 8 * 8) and info["vec"] == vec
        assert info["groups_per_cta"] == min(G, 256) and info["slices"] * info["groups_per_cta"] >= G
        assert info["lanes"] * info["groups_per_cta"] <= 256 and info["pixels_per_cta"] == 8 * info["lanes"]
        assert (info["ranges"] - 1) * info["pixels_per_cta"] < HW <= info["ranges"] * info["pixels_per_cta"]
        assert info["ctas"] == N * info["ranges"] * info["slices"]
        # a function of the shape alone: the batch only multiplies the CTAs
        other = pkg.global_avgpool_nhwc_info(N + 3, H, W, C, pitch)
        assert {k: v for k, v in other.items() if k != "ctas"} == {k: v for k, v in info.items() if k != "ctas"}
    assert accepted > 100 and refused > 100, (accepted, refused)
    big = pkg.global_avgpool_nhwc_info(8, 56, 56, 256)                 # a small batch of large images still spreads
    assert big["ranges"] == 49 and big["ctas"] == 392
    assert pkg.global_avgpool_nhwc_info(1, 1, 1, 2048)["ranges"] == 1
    with pytest.raises(pkg.PcnnError, match="32-bit index range"):
        pkg.global_avgpool_nhwc_info(1, 46341, 46341, 1)
