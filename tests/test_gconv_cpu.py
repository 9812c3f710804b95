"""Host-only checks of the grouped convolution: the references of tests/gconv_ref.py pinned to torch's CPU float64
conv2d(groups=G) and its gradients (the Cg = 1 channel multiplier included), and pcnn_gconv_info over its domain with every
refusal."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gconv_ref as GR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

GROUPINGS = [  # C, K, G: Cg, Kg
    (8, 8, 2),      # 4, 4
    (6, 9, 3),      # 2, 3
    (4, 8, 4),      # 1, 2: a channel multiplier
    (3, 6, 3),      # 1, 2
    (16, 8, 2),     # 8, 4
    (12, 4, 2),     # 6, 2
    (6, 3, 3),      # 2, 1
]
WINDOWS = [(3, 3), (5, 5), (1, 1), (3, 2), (7, 7)]
CASES = [  # N, H, W, C, K, G, R, S, stride, pad_h, pad_w
    (2, 9, 11, C, K, G, R, S, st, ph, pw)
    for (C, K, G) in GROUPINGS
    for (R, S) in WINDOWS
    for st in (1, 2, 3)
    for (ph, pw) in sorted({(0, 0), (R - 1, S - 1), (R // 2, S // 2 if S > 1 else 0)})
    if (C, K, G) in GROUPINGS[:3] or (st == 2 and (R, S) in ((3, 3), (3, 2)))
]


def special(rng, shape):
    a = rng.standard_normal(shape)
    flat = a.reshape(-1)
    for v, n in ((np.nan, 2), (np.inf, 2), (-np.inf, 2), (0.0, 4), (-0.0, 4)):
        flat[rng.choice(flat.size, n, replace=False)] = v
    return a


def nchw(a):
    return torch.from_numpy(np.ascontiguousarray(a)).permute(0, 3, 1, 2)


def torch_w(w):
    return torch.from_numpy(np.ascontiguousarray(w)).permute(0, 3, 1, 2)          # [K][R][S][Cg] -> [K][Cg][R][S]


def nhwc(t):
    return t.permute(0, 2, 3, 1).numpy()


def same(a, b, rtol=0.0, atol=0.0):
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.allclose(a[~np.isnan(a)], b[~np.isnan(b)], rtol=rtol, atol=atol)


@pytest.mark.parametrize("case", CASES, ids=["x".join(map(str, c)) for c in CASES])
def test_references_match_torch_float64(case):
    N, H, W, C, K, G, R, S, st, ph, pw = case
    rng = np.random.default_rng(sum(case))
    x = rng.standard_normal((N, H, W, C))
    w = rng.standard_normal((K, R, S, C // G))
    b = rng.standard_normal(K)
    P, Q = GR.out_size(H, W, R, S, st, ph, pw)
    want = nhwc(F.conv2d(nchw(x), torch_w(w), torch.from_numpy(b), st, (ph, pw), groups=G))
    assert want.shape == (N, P, Q, K)
    assert same(GR.fwd_f64(x, w, G, b, st, ph, pw), want, rtol=1e-12, atol=1e-12)
    assert same(GR.fwd_f64(x, w, G, b, st, ph, pw, act=3), np.maximum(want, 0.0), rtol=1e-12, atol=1e-12)
    # gradients, from torch's autograd
    dy = rng.standard_normal((N, P, Q, K))
    xt, wt = nchw(x).requires_grad_(True), torch_w(w).requires_grad_(True)
    F.conv2d(xt, wt, None, st, (ph, pw), groups=G).backward(nchw(dy))
    assert same(GR.dgrad_f64(dy, w, G, H, W, st, ph, pw), nhwc(xt.grad), rtol=1e-12, atol=1e-12)
    assert same(GR.wgrad_f64(x, dy, G, R, S, st, ph, pw), wt.grad.permute(0, 2, 3, 1).numpy(), rtol=1e-12, atol=1e-12)
    # the float32 replays are the float64 results rounded along the way
    x32, w32, dy32 = x.astype(np.float32), w.astype(np.float32), dy.astype(np.float32)
    assert np.allclose(GR.fwd(x32, w32, G, b.astype(np.float32), st, ph, pw), want, rtol=1e-4, atol=1e-4)
    dx32, terms = GR.dgrad(dy32, w32, G, H, W, st, ph, pw)
    assert np.allclose(dx32, nhwc(xt.grad), rtol=1e-4, atol=1e-4)
    assert np.all(dx32[:, terms == 0].view(np.uint32) == 0)                          # +0 with no term


SPECIAL = [c for c in CASES if c[6:9] in ((3, 3, 1), (3, 3, 2), (3, 2, 3), (1, 1, 2)) and c[3:6] in GROUPINGS[:3]]


@pytest.mark.parametrize("case", SPECIAL, ids=["x".join(map(str, c)) for c in SPECIAL])
def test_special_values_match_torch_float64(case):
    """+-0, +-Inf and NaN in x and dy, and Inf in the filters: taps outside the image multiply +0, so 0 * Inf is NaN, as in torch"""
    N, H, W, C, K, G, R, S, st, ph, pw = case
    rng = np.random.default_rng(7 + sum(case))
    x, w = special(rng, (N, H, W, C)), rng.standard_normal((K, R, S, C // G))
    w[0, 0, 0, 0] = np.inf
    P, Q = GR.out_size(H, W, R, S, st, ph, pw)
    assert same(GR.fwd_f64(x, w, G, None, st, ph, pw), nhwc(F.conv2d(nchw(x), torch_w(w), None, st, (ph, pw), groups=G)),
                rtol=1e-12, atol=1e-12)
    dy = special(rng, (N, P, Q, K))
    gi = torch.nn.grad.conv2d_input((N, C, H, W), torch_w(w), nchw(dy), st, (ph, pw), groups=G)
    assert same(GR.dgrad_f64(dy, w, G, H, W, st, ph, pw), nhwc(gi), rtol=1e-12, atol=1e-12)
    gw = torch.nn.grad.conv2d_weight(nchw(x), (K, C // G, R, S), nchw(dy), st, (ph, pw), groups=G)
    assert same(GR.wgrad_f64(x, dy, G, R, S, st, ph, pw), gw.permute(0, 2, 3, 1).numpy(), rtol=1e-12, atol=1e-12)


def test_info_domain(pkg):
    i = pkg.gconv_info(128, 56, 56, 128, 128, 32, 3, 3, 1, (1, 1))
    assert (i["P"], i["Q"], i["Cg"], i["Kg"], i["vec"], i["kt"]) == (56, 56, 4, 4, 4, 4)
    assert pkg.gconv_info(128, 56, 56, 256, 256, 32, 3, 3, 2, (1, 1))["vec"] == 8
    assert pkg.gconv_info(2, 9, 9, 32, 64, 32, 3, 3)["vec"] == 1                    # channel multiplier: Cg = 1, Kg = 2
    for (C, K, G) in ((8, 8, 2), (64, 128, 32), (32, 64, 32), (384, 384, 8), (1024, 1024, 32), (6, 9, 3), (200, 600, 8), (2048, 64, 2)):
        for (R, S) in WINDOWS:
            if (K // G) * (C // G) * R * S > 36864:
                continue
            for st in (1, 2, 3, 4):
                i = pkg.gconv_info(4, 13, 10, C, K, G, R, S, st, (R - 1, S - 1))
                assert (i["P"], i["Q"]) == GR.out_size(13, 10, R, S, st, R - 1, S - 1)
                Cg, Kg = C // G, K // G
                assert (i["Cg"], i["Kg"]) == (Cg, Kg)
                assert i["vec"] == max(v for v in (1, 2, 4, 8) if Cg % v == 0) and i["kt"] == max(v for v in (1, 2, 4, 8) if Kg % v == 0)
                assert i["fwd_slices"] * i["fwd_tiles_per_cta"] * i["kt"] >= K and i["fwd_tiles_per_cta"] <= 32
                assert i["dgrad_slices"] * i["dgrad_tiles_per_cta"] * i["vec"] >= C and i["dgrad_tiles_per_cta"] <= 32
                assert i["wgrad_items"] == (K // i["kt"]) * R * S * (Cg // i["vec"]) and i["wgrad_item_blocks"] == -(-i["wgrad_items"] // 32)
                M = 4 * i["P"] * i["Q"]
                assert i["ranges"] == -(-M // i["pixels_per_range"]) and i["pixels_per_range"] == i["lanes"] * 64
    # the split depends on the shape alone: the same answer every time, and a larger batch only adds ranges
    a = pkg.gconv_info(128, 28, 28, 256, 256, 32, 3, 3, 1, (1, 1))
    assert a == pkg.gconv_info(128, 28, 28, 256, 256, 32, 3, 3, 1, (1, 1))
    b = pkg.gconv_info(256, 28, 28, 256, 256, 32, 3, 3, 1, (1, 1))
    assert b["pixels_per_range"] == a["pixels_per_range"] and b["ranges"] == 2 * a["ranges"]
    assert a["n_acc"] == 63 + (a["lanes"] - 1) + (-(-a["ranges"] // 8) + 3)
    one = pkg.gconv_info(1, 3, 3, 8, 8, 2, 3, 3, 1, (1, 1))
    assert one["ranges"] == 1 and one["n_acc"] == 1 + 7                      # 9 pixels over 8 lanes: two for lane 0, 8 lanes
    # the largest filters the staging admits: every 1x1 and 3x3 with Cg, Kg <= 64, 5x5 and 7x7 with Cg Kg <= 64
    for (R, S) in ((1, 1), (3, 3)):
        pkg.gconv_info(2, 8, 8, 128, 128, 2, R, S, 1, (R // 2, S // 2))
    for (R, S) in ((5, 5), (7, 7)):
        for (Cg, Kg) in ((8, 8), (1, 64), (64, 1), (2, 32)):
            pkg.gconv_info(2, 8, 8, 2 * Cg, 2 * Kg, 2, R, S, 1, (R // 2, S // 2))


def test_info_independent_of_the_device(pkg):
    """pcnn_gconv_info takes no context: a process that sees no GPU at all gets the same partition"""
    shapes = [(128, 14, 14, 512, 512, 32, 3, 3, 1, (1, 1)), (128, 56, 56, 32, 64, 32, 3, 3, 1, (1, 1)), (3, 9, 7, 12, 4, 2, 5, 5, 3, (4, 0))]
    code = ("import json, pcnn_loader; pkg = pcnn_loader.load(); "
            f"print(json.dumps([pkg.gconv_info(*s) for s in {shapes!r}]))")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, check=True).stdout
    assert json.loads(out) == [pkg.gconv_info(*s) for s in shapes]


REFUSALS = [  # args of gconv_info (N, H, W, C, K, G, R, S, stride, padding), words of the message
    ((0, 8, 8, 8, 8, 2, 3, 3, 1, (0, 0)), "each must be >= 1"),
    ((1, 8, 8, 0, 8, 2, 3, 3, 1, (0, 0)), "each must be >= 1"),
    ((1, 8, 8, 8, 0, 2, 3, 3, 1, (0, 0)), "K >= 1 is required"),
    ((1, 8, 8, 8, 8, 2, 8, 3, 1, (0, 0)), "1 <= R, S <= 7"),
    ((1, 8, 8, 8, 8, 2, 3, 3, 0, (0, 0)), "1 <= stride <= 4"),
    ((1, 8, 8, 8, 8, 2, 3, 3, 5, (0, 0)), "1 <= stride <= 4"),
    ((1, 8, 8, 8, 8, 2, 3, 3, 1, (3, 0)), "0 <= pad_h <= R - 1"),
    ((1, 8, 8, 8, 8, 2, 3, 3, 1, (0, -1)), "0 <= pad_w <= S - 1"),
    ((1, 2, 8, 8, 8, 2, 5, 3, 1, (1, 0)), "H + 2 pad_h >= R"),
    ((1, 8, 1, 8, 8, 2, 3, 3, 1, (0, 0)), "W + 2 pad_w >= S"),
    ((1, 8, 8, 8, 8, 1, 3, 3, 1, (0, 0)), "groups = 1 is a dense convolution: use ConvLayer"),
    ((1, 8, 8, 8, 8, 0, 3, 3, 1, (0, 0)), "G >= 2 is required"),
    ((1, 8, 8, 8, 8, -2, 3, 3, 1, (0, 0)), "G >= 2 is required"),
    ((1, 8, 8, 9, 8, 2, 3, 3, 1, (0, 0)), "C % G == 0 and K % G == 0"),
    ((1, 8, 8, 8, 9, 2, 3, 3, 1, (0, 0)), "C % G == 0 and K % G == 0"),
    ((1, 8, 8, 8, 8, 8, 3, 3, 1, (0, 0)), "use pcnn_dwconv_plan_create"),
    ((1, 8, 8, 256, 256, 2, 3, 3, 1, (1, 1)), "Kg Cg R S <= 36864"),
    ((1, 8, 8, 128, 128, 2, 5, 5, 1, (2, 2)), "Kg Cg R S <= 36864"),
    ((1, 32768, 32768, 8, 8, 2, 3, 3, 1, (0, 0)), "32-bit index range"),
    ((1, 8, 8, 2 ** 26, 2 ** 26, 2 ** 25, 1, 1, 1, (0, 0)), "32-bit index range"),
]


@pytest.mark.parametrize("args,words", REFUSALS, ids=[w for _, w in REFUSALS])
def test_info_refusals(pkg, args, words):
    with pytest.raises(pkg.PcnnError) as e:
        pkg.gconv_info(*args)
    assert "pcnn_gconv_info" in e.value.msg and words in e.value.msg, e.value.msg


def test_layer_refuses_a_wide_activation_backward(pkg):
    """a bias or a ReLU routes the backward through pcnn_conv_bias_act_bwd, which takes K <= 256: the layer refuses a larger K
    before it touches the device"""
    with pytest.raises(pkg.PcnnError) as e:
        pkg.GroupedConvLayer(None, 2, 8, 8, 512, 512, 32, 3, 3, np.zeros((512, 3, 3, 16), np.float32), act=pkg.ACT_RELU)
    assert "K <= 256" in e.value.msg
    with pytest.raises(pkg.PcnnError) as e:
        pkg.GroupedConvLayer(None, 2, 8, 8, 512, 512, 32, 3, 3, np.zeros((512, 3, 3, 16), np.float32), np.zeros(512, np.float32))
    assert "K <= 256" in e.value.msg
