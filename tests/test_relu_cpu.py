"""The ReLU activation without a GPU: the numpy reference of relu_ref.py pinned to torch.relu and threshold_backward in float32
and float64, on NaN, +-0, +-Inf, subnormals, values below bf16's smallest subnormal and exact bf16 rounding ties, and the
exported activation codes."""
import numpy as np
import torch

import relu_ref as RR

TINY = 2.0 ** -133                     # bf16's smallest subnormal
SPECIAL = [0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 1.0, -1.0, 1e-40, -1e-40, 1.4e-45, -1.4e-45, 2.0 ** -126, -(2.0 ** -126),
           TINY, -TINY, TINY / 2, -TINY / 2, 0.75 * TINY, -0.75 * TINY, 1.5 * TINY, 2.0 ** -140, -(2.0 ** -140),
           1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), -(1.0 + 3 * 2.0 ** -8), 0.5 + 2.0 ** -9, 3.4e38, -3.4e38,
           3.39e38, 65504.0, -65504.0]


def values(dtype, rng):
    v = np.concatenate([np.array(SPECIAL, np.float64), rng.standard_normal(2000) * 10.0 ** rng.integers(-45, 38, 2000)])
    return v.astype(dtype)


def same_bits(a, b):
    """identical, except that NaNs compare as NaN (torch and numpy may pick different NaN payloads)"""
    a, b = np.asarray(a), np.asarray(b)
    nan = np.isnan(a)
    if not np.array_equal(nan, np.isnan(b)):
        return False
    u = np.uint32 if a.dtype == np.float32 else np.uint64
    return np.array_equal(a[~nan].view(u), b[~nan].view(u))


def test_forward_matches_torch_relu():
    rng = np.random.default_rng(1)
    for dt in (np.float32, np.float64):
        v = values(dt, rng)
        t = torch.from_numpy(v)
        for want in (torch.relu(t).numpy(), torch.clamp_min(t, 0).numpy()):
            assert same_bits(RR.relu(v), want), dt
        r = RR.relu(v)
        assert np.signbit(r[1]) and not np.signbit(r[0])                 # -0 passes, +0 stays
        assert np.isnan(r[4]) and np.isnan(r[5])                          # NaN passes (fmax would give 0)
        assert r[3] == 0 and not np.signbit(r[3])                         # -Inf gives +0


def test_forward_rounding_matches_torch_bf16(pkg):
    """y = bf16_rn(relu(v)) of fp32 v: the bits of torch.relu(v).to(bfloat16), with one rounding after the ReLU: a negative v never
    becomes -0, a positive v below half of bf16's smallest subnormal becomes +0, ties go to even"""
    rng = np.random.default_rng(2)
    v = values(np.float32, rng)
    got = RR.fwd_bits(pkg, v)
    want = torch.relu(torch.from_numpy(v)).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    nan = np.isnan(v)
    assert np.array_equal(got[~nan], want[~nan])
    assert np.all((got[nan] & 0x7FFF) > 0x7F80)
    f = pkg.bf16_bits_to_f32(got)
    assert not np.any((got == 0x8000) & (v < 0))                         # no -0 from a negative v
    assert f[SPECIAL.index(TINY / 2)] == 0 and f[SPECIAL.index(0.75 * TINY)] == np.float32(TINY)
    assert f[SPECIAL.index(1.5 * TINY)] == np.float32(2 * TINY)          # tie of subnormals to even
    assert f[SPECIAL.index(1.0 + 2.0 ** -8)] == 1.0 and f[SPECIAL.index(1.0 + 3 * 2.0 ** -8)] == np.float32(1.0 + 2.0 ** -6)
    assert f[SPECIAL.index(-(1.0 + 3 * 2.0 ** -8))] == 0


def test_backward_matches_threshold_backward(pkg):
    """dpre = y <= 0 ? +0 : dy on the bf16 values, the bits of dy passed through, as aten.threshold_backward(dy, y, 0)"""
    rng = np.random.default_rng(3)
    n = 4096
    y = np.concatenate([np.array(SPECIAL, np.float32), rng.standard_normal(n - len(SPECIAL)).astype(np.float32)])
    dy = rng.permutation(np.concatenate([np.array(SPECIAL, np.float32), rng.standard_normal(n - len(SPECIAL)).astype(np.float32)]))
    yb, dyb = pkg.f32_to_bf16_bits(y), pkg.f32_to_bf16_bits(dy)
    got = RR.bwd_bits(pkg, yb, dyb)
    for dt in (torch.float32, torch.float64):
        yt = torch.from_numpy(pkg.bf16_bits_to_f32(yb)).to(dt)
        dyt = torch.from_numpy(pkg.bf16_bits_to_f32(dyb)).to(dt)
        want = torch.ops.aten.threshold_backward(dyt, yt, 0).numpy()
        assert same_bits(pkg.bf16_bits_to_f32(got).astype(want.dtype), want), dt
    yf = pkg.bf16_bits_to_f32(yb)
    passed = ~(yf <= 0)
    assert np.array_equal(got[passed], dyb[passed])                    # NaN y included: dy's bits, no arithmetic
    assert np.all(got[~passed] == 0)                                   # +0, never -0, for y <= 0 (y = -0 included)
    assert np.isnan(yf).any() and (yf == 0).any() and np.signbit(yf[yf == 0]).any()


def test_activation_codes_exported(pkg):
    assert (pkg.ACT_NONE, pkg.ACT_SIGMOID, pkg.ACT_RELU) == (0, 1, 3)
    import os
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "pcnn.h")).read()
    for name, v in (("NONE", 0), ("SIGMOID", 1), ("RELU", 3)):
        assert f"#define PCNN_ACT_{name} {v}\n" in header
