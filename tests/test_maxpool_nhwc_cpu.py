"""Host-side parts of the NHWC max pool (no GPU): the numpy reference the GPU tests pin the kernels to agrees with torch's CPU
max_pool2d(return_indices=True) and max_pool2d_with_indices_backward in float32 and float64, ties, NaN, +-Inf, +-0 and all -Inf
windows included; pcnn_maxpool_nhwc_info accepts exactly the stated domain, with torch's output size, and names every rule it
refuses."""
import itertools

import numpy as np
import pytest
import torch

import maxpool_ref as MR


def special_input(rng, shape, dtype):
    """small integers (ties everywhere) with NaN, +-Inf, +-0 sprinkled in, and one image row of -Inf"""
    x = rng.integers(-3, 4, shape).astype(dtype)
    flat = x.reshape(-1)
    for v, frac in ((np.nan, 0.04), (np.inf, 0.03), (-np.inf, 0.08), (0.0, 0.05), (-0.0, 0.05)):
        idx = rng.choice(flat.size, max(1, int(frac * flat.size)), replace=False)
        flat[idx] = v
    x[:, 0] = -np.inf                                        # windows of all -Inf where the window is one row tall
    return x


def torch_pool(x, R, S, st, ph, pw):
    xt = torch.from_numpy(x).permute(0, 3, 1, 2)
    y, idx = torch.nn.functional.max_pool2d(xt, (R, S), st, (ph, pw), return_indices=True)
    return xt, y, idx


CASES = [  # N, H, W, C, R, S, stride, pad_h, pad_w
    (2, 6, 8, 3, 2, 2, 2, 0, 0),
    (2, 7, 9, 4, 3, 3, 2, 1, 1),
    (1, 7, 7, 2, 3, 3, 1, 1, 1),
    (2, 9, 8, 3, 3, 2, 3, 0, 1),       # stride > window: gaps
    (1, 11, 10, 2, 2, 2, 2, 1, 0),
    (1, 14, 14, 2, 7, 7, 7, 3, 0),
    (2, 5, 6, 3, 1, 1, 2, 0, 0),
    (1, 12, 9, 2, 5, 4, 2, 2, 2),
    (3, 1, 9, 2, 1, 3, 1, 0, 1),       # one row: windows of all -Inf
]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("case", CASES, ids=["x".join(map(str, c)) for c in CASES])
def test_reference_matches_torch_cpu(case, dtype):
    N, H, W, C, R, S, st, ph, pw = case
    rng = np.random.default_rng(sum(case))
    ibits = np.uint32 if dtype == np.float32 else np.uint64
    for x in (special_input(rng, (N, H, W, C), dtype), rng.integers(0, 3, (N, H, W, C)).astype(dtype)):
        xt, y, idx = torch_pool(x, R, S, st, ph, pw)
        a = MR.fwd_argmax(x, R, S, st, ph, pw)
        P, Q = MR.out_size(H, W, R, S, st, ph, pw)
        assert tuple(y.shape) == (N, C, P, Q)
        h, w = MR.winner_hw(a, S, st, ph, pw)
        assert np.array_equal(idx.permute(0, 2, 3, 1).numpy(), h * W + w)
        got = MR.gather(x, a, S, st, ph, pw)
        assert np.array_equal(y.permute(0, 2, 3, 1).numpy().view(ibits), got.view(ibits))      # -0 / +0 and NaN bits too
        for dy in (rng.integers(-3, 4, (N, P, Q, C)).astype(dtype), rng.standard_normal((N, P, Q, C)).astype(dtype)):
            want = torch.ops.aten.max_pool2d_with_indices_backward(torch.from_numpy(dy).permute(0, 3, 1, 2), xt, [R, S], [st, st],
                                                                    [ph, pw], [1, 1], False, idx)
            dx, cnt = MR.bwd_sum(dy, a, H, W, R, S, st, ph, pw)
            assert np.array_equal(want.permute(0, 2, 3, 1).numpy(), dx)
            assert np.all(dx[cnt == 0] == 0)
        if st >= R and st >= S:
            assert MR.bwd_sum(np.ones((N, P, Q, C), dtype), a, H, W, R, S, st, ph, pw)[1].max() <= 1


def test_reference_special_windows():
    """the rule on hand-made windows: first maximum of a tie, -0 before +0, last NaN, first element of an all -Inf window"""
    ninf, nan = -np.inf, np.nan
    rows = [[1, 3, 3, 2], [-0.0, 0.0, 0.0, -1], [0.0, -0.0, -0.0, -1], [nan, 5, nan, 7], [ninf, ninf, ninf, ninf], [ninf, 2, ninf, 2]]
    x = np.array(rows, np.float32).reshape(len(rows), 1, 4, 1)
    a = MR.fwd_argmax(x, 1, 4, 1, 0, 0)[:, 0, 0, 0]
    assert list(a) == [1, 0, 0, 2, 0, 1]
    y = MR.gather(x, MR.fwd_argmax(x, 1, 4, 1, 0, 0), 4, 1, 0, 0)[:, 0, 0, 0]
    assert np.signbit(y[1]) and not np.signbit(y[2])
    _, _, idx = torch_pool(x, 1, 4, 1, 0, 0)
    assert list(idx[:, 0, 0, 0].numpy()) == list(a)


def test_reference_bf16_backward(pkg):
    """one term keeps dy's bits (NaN payload included), none gives +0, several round the float32 sum once"""
    x = np.array([[1, 2, 0], [0, 5, 0], [3, 0, 4]], np.float32).reshape(1, 3, 3, 1)
    a = MR.fwd_argmax(x, 2, 2, 1, 0, 0)                     # every window of this 2x2 / 1 picks the 5 in the middle
    assert np.all(a == np.array([3, 2, 1, 0]).reshape(1, 2, 2, 1))
    dy = pkg.f32_to_bf16_bits(np.array([1.0, 2.0 ** -8, 2.0 ** -8, 2.0 ** -8], np.float32)).reshape(1, 2, 2, 1)
    dx = MR.bwd_bf16(pkg, dy, a, 3, 3, 2, 2, 1, 0, 0)
    assert dx[0, 1, 1, 0] == pkg.f32_to_bf16_bits(np.float32(1.0 + 3 * 2.0 ** -8))          # fp32 sum, one rounding
    assert np.all(np.delete(dx.reshape(-1), 4) == 0)
    nan = np.array([0x7FA1], np.uint16).reshape(1, 1, 1, 1)
    a1 = MR.fwd_argmax(np.zeros((1, 2, 2, 1), np.float32), 2, 2, 2, 0, 0)
    assert MR.bwd_bf16(pkg, nan, a1, 2, 2, 2, 2, 2, 0, 0)[0, 0, 0, 0] == 0x7FA1


# ------------------------------------------------------------------------------------------------ pcnn_maxpool_nhwc_info
def domain_refusal(N, H, W, C, R, S, st, ph, pw):
    """the rule of include/pcnn.h a shape breaks first (None: accepted), as the message names it"""
    if min(N, H, W, C) < 1:
        return "each must be >= 1"
    if not (1 <= R <= 7 and 1 <= S <= 7):
        return "1 <= R, S <= 7"
    if not 1 <= st <= 7:
        return "1 <= stride <= 7"
    if not (0 <= ph <= R // 2 and 0 <= pw <= S // 2):
        return "pad_h <= R/2 and 0 <= pad_w <= S/2"
    if H + 2 * ph < R or W + 2 * pw < S:
        return "H + 2 pad_h >= R and W + 2 pad_w >= S"
    return None


def cover_brute(H, R, st, pad, P):
    return max(len([p for p in range(P) if p * st - pad <= h <= p * st - pad + R - 1]) for h in range(H))


def test_info_domain_grid(pkg):
    counts = {"accepted": 0, "refused": 0}
    for R, S, st in itertools.product(range(1, 8), range(1, 8), range(1, 8)):
        for ph, pw in itertools.product(range(R // 2 + 2), range(S // 2 + 2)):
            for H, W in itertools.product((1, 2, 3, 6, 11), (1, 4, 7)):
                C = 3 if (R + S + st) % 2 else 16
                rule = domain_refusal(1, H, W, C, R, S, st, ph, pw)
                try:
                    info = pkg.maxpool_nhwc_info(1, H, W, C, R, S, st, (ph, pw))
                except pkg.PcnnError as e:
                    assert rule is not None and rule in e.msg and "pcnn_maxpool_nhwc_info" in e.msg, (R, S, st, ph, pw, H, W, e.msg)
                    counts["refused"] += 1
                    continue
                assert rule is None, (R, S, st, ph, pw, H, W)
                counts["accepted"] += 1
                P, Q = MR.out_size(H, W, R, S, st, ph, pw)
                assert (info["P"], info["Q"]) == (P, Q)
                assert info["row_pitch"] == (Q * C + 7) // 8 * 8 and info["vec"] == (8 if C % 8 == 0 else 1)
                assert info["cover"] == cover_brute(H, R, st, ph, P) * cover_brute(W, S, st, pw, Q)
                if (H + W) % 5 == 0:                             # torch agrees on the output size
                    y = torch.nn.functional.max_pool2d(torch.zeros(1, 1, H, W), (R, S), st, (ph, pw))
                    assert tuple(y.shape[2:]) == (P, Q)
    assert counts["accepted"] > 1000 and counts["refused"] > 1000, counts


def test_info_refusal_messages(pkg):
    info = pkg.maxpool_nhwc_info
    cases = [
        (lambda: info(0, 4, 4, 8, 2, 2, 2), "each must be >= 1"),
        (lambda: info(1, 4, 0, 8, 2, 2, 2), "each must be >= 1"),
        (lambda: info(1, 4, 4, 0, 2, 2, 2), "each must be >= 1"),
        (lambda: info(1, 9, 9, 8, 8, 2, 2), "1 <= R, S <= 7"),
        (lambda: info(1, 9, 9, 8, 2, 0, 2), "1 <= R, S <= 7"),
        (lambda: info(1, 9, 9, 8, 2, 2, 0), "1 <= stride <= 7"),
        (lambda: info(1, 9, 9, 8, 2, 2, 8), "1 <= stride <= 7"),
        (lambda: info(1, 9, 9, 8, 3, 3, 2, (2, 1)), "pad_h <= R/2"),
        (lambda: info(1, 9, 9, 8, 3, 3, 2, (1, -1)), "pad_h <= R/2"),
        (lambda: info(1, 2, 9, 8, 5, 3, 2, (2, 1)), None),
        (lambda: info(1, 2, 9, 8, 7, 3, 2, (2, 1)), "H + 2 pad_h >= R"),
        (lambda: info(1, 9, 1, 8, 3, 4, 2, (1, 1)), "W + 2 pad_w >= S"),
        (lambda: info(1, 8, 8, 6, 2, 2, 2, row_pitch=20), "row_pitch 20"),          # Q*C = 24
        (lambda: info(1, 8, 8, 6, 2, 2, 2, row_pitch=28), "multiple of 8"),
        (lambda: info(1, 8, 8, 6, 2, 2, 2, image_rows=3), "image_rows 3: 0 (P) or >= P = 4"),
        (lambda: info(1, 8, 8, 6, 2, 2, 2, image_rows=-1), "image_rows -1"),
        (lambda: info(1, 46341, 46341, 8, 2, 2, 2), "32-bit index range"),
    ]
    for fn, msg in cases:
        if msg is None:
            fn()
            continue
        with pytest.raises(pkg.PcnnError, match=msg.replace("(", r"\(").replace(")", r"\)").replace("+", r"\+")):
            fn()
    assert info(1, 8, 8, 6, 2, 2, 2, row_pitch=32, image_rows=7) == dict(P=4, Q=4, row_pitch=32, vec=1, cover=1)
    assert info(1, 8, 8, 6, 2, 2, 2)["row_pitch"] == 24
    assert info(1, 8, 8, 5, 2, 2, 2)["row_pitch"] == 24                              # Q*C = 20 rounded up to 8
    assert info(1, 7, 7, 8, 3, 3, 1, (1, 1))["cover"] == 9 and info(1, 7, 7, 8, 3, 3, 2, (1, 1))["cover"] == 4
    assert info(1, 9, 8, 8, 3, 2, 3)["cover"] == 1
