"""Host-only checks of squeeze-and-excitation: the float64 references of tests/se_ref.py pinned to torch's CPU float64
relu(x * s[:, :, None, None] + r) and its autograd, the whole block's decomposition (gate pass, fc2 and fc1 backward, input pass with
dpool) pinned to torch's autograd of x * sigmoid(fc2(relu(fc1(x.mean((2, 3)))))), the float32 replays against float64, the
partition query pcnn_se_scale_nhwc_info, and the refusals that need no GPU."""
import numpy as np
import pytest
import torch

import se_ref as SR

SHAPES = [(2, 1, 1, 3), (3, 7, 7, 8), (2, 5, 6, 6), (2, 4, 4, 16)]


def nchw(a):
    return torch.from_numpy(np.ascontiguousarray(a.transpose(0, 3, 1, 2)))


def nhwc(t):
    return t.detach().permute(0, 2, 3, 1).numpy()


@pytest.mark.parametrize("act", [0, 3])
@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
def test_scale_against_torch(shape, act):
    N, H, W, C = shape
    rng = np.random.default_rng(sum(shape) + act)
    x, r, dy, dy2 = (rng.standard_normal(shape) for _ in range(4))
    s = rng.uniform(0, 1, (N, C))
    for with_r, with_dy2 in ((False, False), (True, True), (True, False)):
        xt, st = nchw(x).requires_grad_(True), torch.from_numpy(s).requires_grad_(True)
        rt = nchw(r).requires_grad_(True) if with_r else None
        v = xt * st[:, :, None, None] + (rt if with_r else 0.0)
        yt = torch.relu(v) if act == 3 else v
        y = SR.fwd(x, s, r if with_r else None, act)
        np.testing.assert_allclose(y, nhwc(yt), rtol=1e-14, atol=1e-14)
        t = dy + dy2 if with_dy2 else dy
        yt.backward(nchw(t))
        g, ds = SR.gate64(x, dy, y, dy2 if with_dy2 else None, act)
        np.testing.assert_allclose(ds, st.grad.numpy(), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(SR.dx(g, s), nhwc(xt.grad), rtol=1e-14, atol=1e-14)
        if with_r:
            np.testing.assert_allclose(g, nhwc(rt.grad), rtol=1e-14, atol=1e-14)


@pytest.mark.parametrize("act", [0, 3])
@pytest.mark.parametrize("shape", [(4, 5, 5, 16), (3, 7, 7, 24), (2, 3, 2, 8)], ids=["4x5x5x16", "3x7x7x24", "2x3x2x8"])
def test_block_decomposition(shape, act):
    """the layer's backward order gives torch's autograd of the whole block, the squeeze branch's gradient included"""
    N, H, W, C = shape
    hid = 8
    rng = np.random.default_rng(C + act)
    x, r, dy = rng.standard_normal(shape), rng.standard_normal(shape), rng.standard_normal(shape)
    w1, b1 = rng.standard_normal((hid, C)) / np.sqrt(C), rng.standard_normal(hid) * 0.1
    w2, b2 = rng.standard_normal((C, hid)) / np.sqrt(hid), rng.standard_normal(C) * 0.1
    f = SR.block_fwd64(x, w1, b1, w2, b2, r, act)
    got = SR.block_bwd64(x, f, w1, w2, dy, act=act)
    T = {k: torch.from_numpy(v).requires_grad_(True) for k, v in dict(w1=w1, b1=b1, w2=w2, b2=b2).items()}
    xt, rt = nchw(x).requires_grad_(True), nchw(r).requires_grad_(True)
    a = torch.relu(xt.mean((2, 3)) @ T["w1"].T + T["b1"])
    st = torch.sigmoid(a @ T["w2"].T + T["b2"])
    v = xt * st[:, :, None, None] + rt
    yt = torch.relu(v) if act == 3 else v
    np.testing.assert_allclose(f["y"], nhwc(yt), rtol=1e-13, atol=1e-13)
    yt.backward(nchw(dy))
    np.testing.assert_allclose(got["dx"], nhwc(xt.grad), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(got["g"], nhwc(rt.grad), rtol=1e-12, atol=1e-12)
    for k in ("w1", "b1", "w2", "b2"):
        np.testing.assert_allclose(got["d" + k], T[k].grad.numpy(), rtol=1e-11, atol=1e-12)
    # without the squeeze branch's gradient (dpool) dx is wrong: the check above can tell
    wrong = SR.dx(got["g"], f["s"])
    assert np.max(np.abs(wrong - nhwc(xt.grad))) > 1e-3


def test_replays_against_float64(pkg):
    """the float32 replays (what the device must match bit for bit) within float32 rounding of float64"""
    N, H, W, C = 3, 9, 7, 16
    info = pkg.se_scale_nhwc_info(N, H, W, C)
    rng = np.random.default_rng(5)
    q = lambda a: SR.bf16(np.asarray(a, np.float32))
    x, r, dy, dy2 = (q(rng.standard_normal((N, H, W, C))) for _ in range(4))
    s, dpool = q(rng.uniform(0, 1, (N, C))), q(rng.standard_normal((N, C)))
    y32 = SR.fwd(x, s, r, 3)
    y64 = SR.fwd(x.astype(np.float64), s.astype(np.float64), r.astype(np.float64), 3)
    assert np.all(np.abs(y32 - y64) <= 2 ** -23 * (np.abs(x * s[:, None, None, :]) + np.abs(y64)))
    g = SR.gate_g(dy, SR.bf16(y32), dy2, 3)
    g64, ds64 = SR.gate64(x.astype(np.float64), dy.astype(np.float64), y32.astype(np.float64), dy2.astype(np.float64), 3)
    assert np.all((g == 0) | (np.abs(g - g64) <= 2 ** -8 * np.abs(g64)))
    ds = SR.gate_ds(g, x, info)
    bound = 2 * info["n_acc"] * 2 ** -24 * (np.abs(g.astype(np.float64) * x).sum(axis=(1, 2)))
    assert np.all(np.abs(ds - (g.astype(np.float64) * x).sum(axis=(1, 2))) <= bound)
    d32 = SR.dx(g, s, dpool, H * W)
    d64 = SR.dx(g.astype(np.float64), s.astype(np.float64), dpool.astype(np.float64), H * W)
    assert np.all(np.abs(d32 - d64) <= 2 ** -23 * (np.abs(g * s[:, None, None, :]) + np.abs(dpool / (H * W))[:, None, None, :] + 1e-30))
    assert SR.gate_ds(g, x, info).tobytes() == ds.tobytes()


def test_bf16_rounding(pkg):
    v = np.array([1.0, 1.00390625, 1.01171875, -2.5, 3.4e38, np.inf, -np.inf, 0.0, -0.0, 1e-40, np.nan], np.float32)
    v = np.concatenate([v, np.random.default_rng(1).standard_normal(1000).astype(np.float32)])
    got = SR.bf16(v)
    want = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(v))
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.array_equal(got[~np.isnan(got)].view(np.uint32), want[~np.isnan(want)].view(np.uint32))


INFO_SHAPES = [(N, H, W, C) for N in (1, 3, 128) for H, W in ((1, 1), (7, 7), (56, 56), (3, 5)) for C in (1, 3, 6, 8, 16, 64, 256, 320, 2048)]


def test_info(pkg):
    """the gate pass's partition is the global average pool's, with n_acc its longest fp32 addition chain"""
    for N, H, W, C in INFO_SHAPES:
        got = pkg.se_scale_nhwc_info(N, H, W, C)
        gap = pkg.global_avgpool_nhwc_info(N, H, W, C)
        for k in ("vec", "groups_per_cta", "slices", "lanes", "pixels_per_cta", "ranges", "ctas"):
            assert got[k] == gap[k], (N, H, W, C, k)
        HW = H * W
        assert got["vec"] == (8 if C % 8 == 0 else 1)
        lane_px = min(8, -(-HW // got["lanes"]))
        assert got["n_acc"] == (lane_px - 1) + (min(got["lanes"], HW) - 1) + (got["ranges"] - 1)
    assert pkg.se_scale_nhwc_info(128, 56, 56, 64)["ranges"] == 13
    assert pkg.se_scale_nhwc_info(2, 7, 7, 2048)["ranges"] == 7


def test_info_matches_replay_order(pkg):
    """a sum whose order matters: the replay in the reported order differs from numpy's own sum order"""
    N, H, W, C = 1, 56, 56, 8
    info = pkg.se_scale_nhwc_info(N, H, W, C)
    p = (np.random.default_rng(3).standard_normal((N, H, W, C)) * 1e3).astype(np.float32)
    a = SR.ordered_sum(p, info)
    seq = np.zeros((N, C), np.float32)
    for px in p.reshape(N, H * W, C).transpose(1, 0, 2):
        seq = seq + px
    assert not np.array_equal(a, seq)
    np.testing.assert_allclose(a, p.astype(np.float64).sum(axis=(1, 2)), rtol=1e-4, atol=1.0)


def test_info_refusals(pkg):
    cases = [((0, 7, 7, 8), "pcnn_se_scale_nhwc_info: N = 0, H = 7, W = 7, C = 8: each must be >= 1"),
             ((2, 0, 7, 8), "each must be >= 1"), ((2, 7, 7, 0), "each must be >= 1"),
             ((2, 46341, 46341, 1), "pcnn_se_scale_nhwc_info: one 46341x46341x1 image exceeds the 32-bit index range"),
             ((2, 4096, 4096, 128), "32-bit index range")]
    for shape, msg in cases:
        with pytest.raises(pkg.PcnnError, match=msg):
            pkg.se_scale_nhwc_info(*shape)


def test_layer_refusals(pkg):
    """SqueezeExcitationLayer refuses what its linear layers cannot hold before it touches the engine"""
    w = np.zeros(1, np.float32)
    cases = [(dict(C=16, hidden=12), "hidden = 12: .*hidden % 8 == 0"), (dict(C=300, hidden=8), "C = 300"),
             (dict(C=16, hidden=264), "hidden = 264"), (dict(C=16, hidden=0), "hidden = 0"),
             (dict(C=16, hidden=8, act=1), "act 1: 0 \\(none\\) or 3 \\(ReLU\\)")]
    for kw, msg in cases:
        act = kw.pop("act", 0)
        with pytest.raises(pkg.PcnnError, match=msg):
            pkg.SqueezeExcitationLayer(None, 2, 4, 4, kw["C"], kw["hidden"], w, w, w, w, act=act)
