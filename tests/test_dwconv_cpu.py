"""Host-only checks of the depthwise convolution: the references of tests/dwconv_ref.py pinned to torch's CPU float64
conv2d(groups=C) and its gradients, and pcnn_dwconv_info over its domain with every refusal."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dwconv_ref as DR

WINDOWS = [(3, 3), (5, 5), (7, 7), (1, 1), (3, 2)]
CASES = [  # N, H, W, C, R, S, stride, pad_h, pad_w
    (N, H, W, C, R, S, st, ph, pw)
    for (R, S) in WINDOWS
    for st in (1, 2, 3, 4)
    for (ph, pw) in sorted({(0, 0), (R - 1, S - 1), (R // 2, S // 2), (min(1, R - 1), 0)})
    for (N, H, W, C) in ((2, 9, 11, 3),)
]


def special(rng, shape):
    a = rng.standard_normal(shape)
    flat = a.reshape(-1)
    for v, n in ((np.nan, 2), (np.inf, 2), (-np.inf, 2), (0.0, 4), (-0.0, 4)):
        flat[rng.choice(flat.size, n, replace=False)] = v
    return a


def torch_conv(x, w, b, st, ph, pw):
    xt = torch.from_numpy(x).permute(0, 3, 1, 2)
    wt = torch.from_numpy(w)[:, None]
    return F.conv2d(xt, wt, None if b is None else torch.from_numpy(b), st, (ph, pw), groups=x.shape[3]).permute(0, 2, 3, 1).numpy()


def same(a, b, rtol=0.0, atol=0.0):
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.allclose(a[~np.isnan(a)], b[~np.isnan(b)], rtol=rtol, atol=atol)


@pytest.mark.parametrize("case", CASES, ids=["x".join(map(str, c)) for c in CASES])
def test_references_match_torch_float64(case):
    N, H, W, C, R, S, st, ph, pw = case
    if H + 2 * ph < R or W + 2 * pw < S:
        pytest.skip("window does not fit")
    rng = np.random.default_rng(sum(case))
    x = rng.standard_normal((N, H, W, C))
    w = rng.standard_normal((C, R, S))
    b = rng.standard_normal(C)
    P, Q = DR.out_size(H, W, R, S, st, ph, pw)
    want = torch_conv(x, w, b, st, ph, pw)
    assert want.shape == (N, P, Q, C)
    assert same(DR.fwd_f64(x, w, b, st, ph, pw), want, rtol=1e-12, atol=1e-12)
    relu = DR.fwd_f64(x, w, b, st, ph, pw, act=3)
    assert same(relu, np.maximum(want, 0.0), rtol=1e-12, atol=1e-12)
    # gradients, from torch's autograd
    dy = rng.standard_normal((N, P, Q, C))
    xt = torch.from_numpy(x).permute(0, 3, 1, 2).requires_grad_(True)
    wt = torch.from_numpy(w)[:, None].requires_grad_(True)
    F.conv2d(xt, wt, None, st, (ph, pw), groups=C).backward(torch.from_numpy(dy).permute(0, 3, 1, 2))
    assert same(DR.dgrad_f64(dy, w, H, W, st, ph, pw), xt.grad.permute(0, 2, 3, 1).numpy(), rtol=1e-12, atol=1e-12)
    assert same(DR.wgrad_f64(x, dy, R, S, st, ph, pw), wt.grad[:, 0].numpy(), rtol=1e-12, atol=1e-12)
    gi = torch.nn.grad.conv2d_input(xt.shape, wt.detach(), torch.from_numpy(dy).permute(0, 3, 1, 2), st, (ph, pw), groups=C)
    assert same(DR.dgrad_f64(dy, w, H, W, st, ph, pw), gi.permute(0, 2, 3, 1).numpy(), rtol=1e-12, atol=1e-12)
    # the float32 replays are the float64 results rounded along the way
    x32, w32, dy32 = x.astype(np.float32), w.astype(np.float32), dy.astype(np.float32)
    assert np.allclose(DR.fwd(x32, w32, b.astype(np.float32), st, ph, pw), want, rtol=1e-4, atol=1e-4)
    dx32, terms = DR.dgrad(dy32, w32, H, W, st, ph, pw)
    assert np.allclose(dx32, xt.grad.permute(0, 2, 3, 1).numpy(), rtol=1e-4, atol=1e-4)
    assert np.all(dx32[:, terms == 0].view(np.uint32) == 0)                          # +0 with no term


@pytest.mark.parametrize("case", [c for c in CASES if c[4:7] in ((3, 3, 1), (3, 3, 2), (5, 5, 1), (3, 2, 3), (1, 1, 4))],
                         ids=lambda c: "x".join(map(str, c)))
def test_special_values_match_torch_float64(case):
    """+-0, +-Inf and NaN in x, and Inf in the filters: taps outside the image multiply +0, so 0 * Inf is NaN, as in torch"""
    N, H, W, C, R, S, st, ph, pw = case
    rng = np.random.default_rng(7 + sum(case))
    x, w = special(rng, (N, H, W, C)), rng.standard_normal((C, R, S))
    w[0, 0, 0] = np.inf
    P, Q = DR.out_size(H, W, R, S, st, ph, pw)
    assert same(DR.fwd_f64(x, w, None, st, ph, pw), torch_conv(x, w, None, st, ph, pw), rtol=1e-12, atol=1e-12)
    dy = special(rng, (N, P, Q, C))
    xt = torch.zeros((N, C, H, W), dtype=torch.float64)
    gi = torch.nn.grad.conv2d_input(xt.shape, torch.from_numpy(w)[:, None], torch.from_numpy(dy).permute(0, 3, 1, 2), st, (ph, pw),
                                    groups=C)
    assert same(DR.dgrad_f64(dy, w, H, W, st, ph, pw), gi.permute(0, 2, 3, 1).numpy(), rtol=1e-12, atol=1e-12)
    gw = torch.nn.grad.conv2d_weight(torch.from_numpy(x).permute(0, 3, 1, 2), (C, 1, R, S), torch.from_numpy(dy).permute(0, 3, 1, 2), st,
                                     (ph, pw), groups=C)
    assert same(DR.wgrad_f64(x, dy, R, S, st, ph, pw), gw[:, 0].numpy(), rtol=1e-12, atol=1e-12)


def test_info_domain(pkg):
    info = pkg.dwconv_info(128, 112, 112, 96, 3, 3, 2, (1, 1))
    assert (info["P"], info["Q"], info["vec"]) == (56, 56, 8)
    assert pkg.dwconv_info(2, 9, 9, 6, 3, 3)["vec"] == 1
    for C in (1, 3, 6, 8, 24, 64, 144, 256, 320, 960, 2048, 1001):
        for (R, S) in WINDOWS:
            for st in (1, 2, 3, 4):
                i = pkg.dwconv_info(4, 13, 10, C, R, S, st, (R - 1, S - 1))
                assert (i["P"], i["Q"]) == DR.out_size(13, 10, R, S, st, R - 1, S - 1)
                G = C // i["vec"]
                assert i["slices"] * i["groups_per_cta"] >= G and i["groups_per_cta"] <= 32
                M = 4 * i["P"] * i["Q"]
                assert i["ranges"] == -(-M // i["pixels_per_range"]) and i["pixels_per_range"] == i["lanes"] * 16
    # the split depends on the shape alone: the same answer every time, and a larger batch only adds ranges
    a = pkg.dwconv_info(128, 56, 56, 144, 3, 3, 1, (1, 1))
    assert a == pkg.dwconv_info(128, 56, 56, 144, 3, 3, 1, (1, 1))
    b = pkg.dwconv_info(256, 56, 56, 144, 3, 3, 1, (1, 1))
    assert b["pixels_per_range"] == a["pixels_per_range"] and b["ranges"] == 2 * a["ranges"]
    assert a["n_acc"] == 15 + (a["lanes"] - 1) + (-(-a["ranges"] // 8) + 3)
    one = pkg.dwconv_info(1, 3, 3, 8, 3, 3, 1, (1, 1))
    assert one["ranges"] == 1 and one["n_acc"] == 0 + 8                        # 9 pixels over 32 lanes: one pixel each, 9 lanes


REFUSALS = [  # args of dwconv_info (N, H, W, C, R, S, stride, padding), words of the message
    ((0, 8, 8, 8, 3, 3, 1, (0, 0)), "each must be >= 1"),
    ((1, 0, 8, 8, 3, 3, 1, (0, 0)), "each must be >= 1"),
    ((1, 8, 0, 8, 3, 3, 1, (0, 0)), "each must be >= 1"),
    ((1, 8, 8, 0, 3, 3, 1, (0, 0)), "each must be >= 1"),
    ((1, 8, 8, 8, 8, 3, 1, (0, 0)), "1 <= R, S <= 7"),
    ((1, 8, 8, 8, 3, 0, 1, (0, 0)), "1 <= R, S <= 7"),
    ((1, 8, 8, 8, 3, 3, 0, (0, 0)), "1 <= stride <= 4"),
    ((1, 8, 8, 8, 3, 3, 5, (0, 0)), "1 <= stride <= 4"),
    ((1, 8, 8, 8, 3, 3, 1, (3, 0)), "0 <= pad_h <= R - 1"),
    ((1, 8, 8, 8, 3, 3, 1, (0, -1)), "0 <= pad_w <= S - 1"),
    ((1, 2, 8, 8, 5, 3, 1, (1, 0)), "H + 2 pad_h >= R"),
    ((1, 8, 1, 8, 3, 3, 1, (0, 0)), "W + 2 pad_w >= S"),
    ((1, 32768, 32768, 8, 3, 3, 1, (0, 0)), "32-bit index range"),
    ((1, 1, 1, 50000000, 7, 7, 1, (3, 3)), "32-bit index range"),
]


@pytest.mark.parametrize("args,words", REFUSALS)
def test_info_refusals(pkg, args, words):
    with pytest.raises(pkg.PcnnError) as e:
        pkg.dwconv_info(*args)
    assert "pcnn_dwconv_info" in e.value.msg and words in e.value.msg, e.value.msg
