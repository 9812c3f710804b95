"""Host-side parts of group normalization (no GPU): the float64 references of groupnorm_ref.py agree with
torch.nn.functional.group_norm followed by the residual add and every activation code, and with torch's autograd through all of
them; at G = C they are instance_norm with affine parameters and at G = 1 layer_norm over (C, H, W); the float32 replays stay
within bf16 rounding of them; pcnn_groupnorm_nhwc_info accepts exactly the stated domain, names every rule it refuses, and gives
a partition that does not change with N."""
import numpy as np
import pytest
import torch

import bnact_ref as BA
import groupnorm_ref as GR

F = torch.nn.functional
TACT = {0: lambda v: v, 3: torch.relu, 4: F.silu, 5: F.hardswish, 6: F.relu6}
ACTS = [0, 3, 4, 5, 6]


def nchw(a):
    """[N][HW][C] numpy -> [N][C][HW][1] float64 torch"""
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float64).transpose(0, 2, 1))).unsqueeze(-1)


def nhwc(t):
    return t.squeeze(-1).permute(0, 2, 1).detach().numpy()


def operands(rng, N, HW, C, with_r, with_dy2):
    x = rng.standard_normal((N, HW, C)) * rng.uniform(0.5, 3, C) + rng.uniform(-4, 4, C)
    gamma, beta = rng.uniform(0.5, 1.5, C), rng.uniform(-0.5, 0.5, C)
    r = rng.standard_normal((N, HW, C)) if with_r else None
    dy = rng.standard_normal((N, HW, C))
    dy2 = rng.standard_normal((N, HW, C)) if with_dy2 else None
    return x, gamma, beta, r, dy, dy2


def torch_block(x, gamma, beta, G, r, dy, dy2, act, eps, norm=None):
    """act(norm(x) + r) in float64 with autograd; norm defaults to F.group_norm(., G, gamma, beta, eps).  Returns y and the
    gradients of x, gamma, beta and r for the incoming dy + dy2."""
    xt = nchw(x).requires_grad_(True)
    gt = torch.from_numpy(np.asarray(gamma, np.float64)).requires_grad_(True)
    bt = torch.from_numpy(np.asarray(beta, np.float64)).requires_grad_(True)
    rt = nchw(r).requires_grad_(True) if r is not None else None
    v = F.group_norm(xt, G, gt, bt, eps) if norm is None else norm(xt, gt, bt)
    if rt is not None:
        v = v + rt
    y = TACT[act](v)
    t = nchw(dy) + (0 if dy2 is None else nchw(dy2))
    y.backward(t)
    return nhwc(y), nhwc(xt.grad), gt.grad.numpy(), bt.grad.numpy(), (nhwc(rt.grad) if rt is not None else None)


SHAPES = [(1, 1, 2, 1), (2, 7, 6, 3), (3, 49, 8, 4), (2, 16, 16, 8), (1, 9, 12, 12), (2, 25, 32, 1), (1, 4, 64, 32)]


@pytest.mark.parametrize("with_dy2", [False, True])
@pytest.mark.parametrize("with_r", [False, True])
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("N,HW,C,G", SHAPES, ids=[f"N{n}-HW{h}-C{c}-G{g}" for n, h, c, g in SHAPES])
def test_references_match_torch(N, HW, C, G, act, with_r, with_dy2):
    """fwd_f64 and bwd_f64 = torch's float64 group_norm (+ r) (+ act) and its autograd: y, dx, dgamma, dbeta and dr (= g)"""
    rng = np.random.default_rng(N * 1009 + HW * 31 + C * 7 + G + 100 * act + 2 * with_r + with_dy2)
    x, gamma, beta, r, dy, dy2 = operands(rng, N, HW, C, with_r, with_dy2)
    y, v, mean, var = GR.fwd_f64(x, gamma, beta, G, r, act)
    dx, dgamma, dbeta, g, A, B = GR.bwd_f64(x, gamma, beta, G, dy, dy2, r, act)
    yt, dxt, dgt, dbt, drt = torch_block(x, gamma, beta, G, r, dy, dy2, act, 1e-5)
    assert np.allclose(y, yt, rtol=1e-12, atol=1e-12)
    assert np.allclose(dx, dxt, rtol=1e-9, atol=1e-10)
    assert np.allclose(dgamma, dgt, rtol=1e-10, atol=1e-10) and np.allclose(dbeta, dbt, rtol=1e-10, atol=1e-10)
    if with_r:
        assert np.allclose(g, drt, rtol=1e-12, atol=1e-12)
    xg = GR.group_view(x, G)
    assert np.allclose(mean, xg.mean(2)) and np.allclose(var, xg.var(2))
    # A and B are the group sums of gamma g and gamma g xhat
    xhat = (x - GR.per_channel(mean, C)) / np.sqrt(GR.per_channel(var, C) + 1e-5)
    assert np.allclose(A, GR.group_view(gamma * g, G).sum(2)) and np.allclose(B, GR.group_view(gamma * g * xhat, G).sum(2))


@pytest.mark.parametrize("act", ACTS)
def test_g_equal_c_is_instance_norm(act):
    """G = C: F.instance_norm with affine parameters (use_input_stats), forward and autograd"""
    rng = np.random.default_rng(40 + act)
    N, HW, C = 3, 20, 6
    x, gamma, beta, r, dy, dy2 = operands(rng, N, HW, C, True, True)
    norm = lambda xt, gt, bt: F.instance_norm(xt, weight=gt, bias=bt, eps=1e-5)
    yt, dxt, dgt, dbt, _ = torch_block(x, gamma, beta, C, r, dy, dy2, act, 1e-5, norm)
    y = GR.fwd_f64(x, gamma, beta, C, r, act)[0]
    dx, dgamma, dbeta = GR.bwd_f64(x, gamma, beta, C, dy, dy2, r, act)[:3]
    assert np.allclose(y, yt, rtol=1e-12, atol=1e-12) and np.allclose(dx, dxt, rtol=1e-9, atol=1e-10)
    assert np.allclose(dgamma, dgt, rtol=1e-10) and np.allclose(dbeta, dbt, rtol=1e-10)


@pytest.mark.parametrize("act", ACTS)
def test_g_one_is_layer_norm(act):
    """G = 1: F.layer_norm over (C, H, W) with gamma and beta expanded over the pixels, forward and autograd"""
    rng = np.random.default_rng(50 + act)
    N, HW, C = 2, 15, 5
    x, gamma, beta, r, dy, dy2 = operands(rng, N, HW, C, True, False)

    def norm(xt, gt, bt):
        return F.layer_norm(xt, (C, HW, 1), gt[:, None, None].expand(C, HW, 1), bt[:, None, None].expand(C, HW, 1), 1e-5)

    yt, dxt, dgt, dbt, _ = torch_block(x, gamma, beta, 1, r, dy, dy2, act, 1e-5, norm)
    y = GR.fwd_f64(x, gamma, beta, 1, r, act)[0]
    dx, dgamma, dbeta = GR.bwd_f64(x, gamma, beta, 1, dy, dy2, r, act)[:3]
    assert np.allclose(y, yt, rtol=1e-12, atol=1e-12) and np.allclose(dx, dxt, rtol=1e-9, atol=1e-10)
    assert np.allclose(dgamma, dgt, rtol=1e-10) and np.allclose(dbeta, dbt, rtol=1e-10)


@pytest.mark.parametrize("act", ACTS)
def test_replays_within_rounding_of_float64(pkg, act):
    """fwd_bits, grad_bits and dx_bits, fed the float64 statistics and group sums rounded to fp32, stay within a few bf16 ulps
    (plus the fp32 cancellation of dx) of fwd_f64 and bwd_f64"""
    rng = np.random.default_rng(60 + act)
    N, HW, C, G = 2, 30, 12, 3
    x, gamma, beta, r, dy, dy2 = operands(rng, N, HW, C, True, True)
    xb, rb, dyb, dy2b = (pkg.f32_to_bf16_bits(a.astype(np.float32)) for a in (x, r, dy, dy2))
    f = lambda b: pkg.bf16_bits_to_f32(b).astype(np.float64)
    x, r, dy, dy2 = f(xb), f(rb), f(dyb), f(dy2b)
    gamma, beta = gamma.astype(np.float32), beta.astype(np.float32)
    y64, v64, mean, var = GR.fwd_f64(x, gamma, beta, G, r, act)
    rstd = (1 / np.sqrt(var + np.float64(np.float32(1e-5)))).astype(np.float32)
    yb = GR.fwd_bits(pkg, xb, gamma, beta, mean.astype(np.float32), rstd, rb, act)
    with np.errstate(invalid="ignore"):
        assert np.all(np.abs(f(yb) - y64) <= 2 ** -7 * np.abs(y64) + 1e-5)
    gb = GR.grad_bits(pkg, xb, gamma, beta, mean.astype(np.float32), rstd, dyb, dy2b, rb, act, yb)
    dx64, _, _, g64, A, B = GR.bwd_f64(x, gamma, beta, G, dy, dy2, r, act)
    assert np.all(np.abs(f(gb) - g64) <= 2 ** -7 * np.abs(g64) + 2 ** -7 * np.abs(dy + dy2).max() * (act in BA.CODES) + 1e-6)
    # dx from the exact g bits: float64 with those g equals the replay within bf16 rounding and fp32 cancellation
    g_exact = f(gb)
    rs64 = GR.per_channel(rstd.astype(np.float64), C)
    xh = (x - GR.per_channel(mean, C)) * rs64
    A64, B64 = GR.group_view(gamma * g_exact, G).sum(2), GR.group_view(gamma * g_exact * xh, G).sum(2)
    Mg = HW * (C // G)
    ref = ((gamma * g_exact - GR.per_channel(A64, C) / Mg) - xh * GR.per_channel(B64, C) / Mg) * rs64
    dxb = GR.dx_bits(pkg, xb, gb, gamma, mean.astype(np.float32), rstd, np.stack([A64, B64]).astype(np.float32))
    scale = (np.abs(gamma * g_exact).max() + np.abs(xh).max() * np.abs(B64).max() / Mg) * rs64.max()
    assert np.all(np.abs(f(dxb) - ref) <= 2 ** -7 * np.abs(ref) + 1e-5 * scale)


# ------------------------------------------------------------------------------------------------ the info query
def refusal(pkg, N, HW, C, G):
    with pytest.raises(pkg.PcnnError) as e:
        pkg.groupnorm_nhwc_info(N, HW, C, G)
    assert e.value.fn == "pcnn_groupnorm_nhwc_info"
    return e.value.msg


def test_info_domain(pkg):
    """exactly N >= 1, HW >= 1, 1 <= C <= 2048, 1 <= G <= C with C % G == 0 are accepted; each refusal names its rule"""
    for N, HW, C, G in [(1, 1, 1, 1), (1, 1, 2048, 2048), (1, 1, 2048, 1), (128, 3136, 64, 32), (3, 7, 6, 3), (2, 65536, 32, 8)]:
        pkg.groupnorm_nhwc_info(N, HW, C, G)
    assert "N >= 1" in refusal(pkg, 0, 1, 8, 1) and "N = 0" in refusal(pkg, 0, 1, 8, 1)
    assert "H * W >= 1" in refusal(pkg, 1, 0, 8, 1) and "H * W >= 1" in refusal(pkg, 1, -5, 8, 1)
    for C in (0, -1, 2049, 4096):
        assert "1 <= C <= 2048" in refusal(pkg, 1, 4, C, 1)
    for C, G in [(8, 0), (8, 16), (8, 3), (6, 4), (2048, 3), (8, -1)]:
        assert "C % G == 0" in refusal(pkg, 1, 4, C, G) and "1 <= G <= C" in refusal(pkg, 1, 4, C, G)
    assert "exceed the grid" in refusal(pkg, 1 << 30, 1 << 20, 8, 1)
    assert pkg.lib().pcnn_groupnorm_nhwc_info(1, 1, 8, 1, None) != 0
    # every divisor G of C is accepted, every other G refused
    for C in (1, 3, 6, 8, 12, 64, 320):
        for G in range(1, C + 2):
            if C % G == 0 and G <= C:
                pkg.groupnorm_nhwc_info(2, 5, C, G)
            else:
                refusal(pkg, 2, 5, C, G)


CASES = [(1, 7), (49, 8), (784, 16), (3136, 64), (3136, 32), (784, 256), (49, 320), (1, 2048), (16384, 64), (65536, 32), (49, 3),
         (784, 6), (7, 1), (3136, 2046)]


@pytest.mark.parametrize("HW,C", CASES, ids=[f"HW{h}-C{c}" for h, c in CASES])
def test_info_partition_does_not_change_with_n(pkg, HW, C):
    """the vector width, slices, lanes, pixels per range and ranges depend on (HW, C) (and G not at all): the same for every N and
    every G; the grids scale with N; the slices cover the channels, the ranges the pixels"""
    base = pkg.groupnorm_nhwc_info(1, HW, C, 1)
    keys = ("vec", "groups_per_cta", "slices", "lanes", "pixels_per_range", "ranges", "n_acc_group")
    for N in (1, 2, 3, 128):
        for G in {1, C, *[g for g in (2, 4, 8, 32) if C % g == 0]}:
            info = pkg.groupnorm_nhwc_info(N, HW, C, G)
            assert all(info[k] == base[k] for k in keys), (N, G, info, base)
            assert info["ctas"] == N * base["ranges"] * base["slices"] and info["slots"] == N * base["ranges"]
            assert info["group_ctas"] == -(-N * G // 8)
            assert info["n_acc"] == 8 + base["lanes"] + -(-N * base["ranges"] // 8) + 3
    vec = 8 if C % 8 == 0 else 1
    assert base["vec"] == vec and base["groups_per_cta"] == min(C // vec, 256 // vec)
    assert base["slices"] * base["groups_per_cta"] * vec >= C > (base["slices"] - 1) * base["groups_per_cta"] * vec
    assert base["lanes"] == 256 // base["groups_per_cta"] and base["pixels_per_range"] == 8 * base["lanes"]
    assert base["ranges"] == -(-HW // base["pixels_per_range"])


def test_benchmark_shapes_fill_the_machine(pkg):
    """the four conv_bench gn shapes run several ranges per image and more CTAs than an H100's 132 SMs"""
    for N, HW, C, G in [(128, 3136, 64, 32), (8, 16384, 64, 32), (2, 65536, 32, 8), (16, 784, 256, 256)]:
        info = pkg.groupnorm_nhwc_info(N, HW, C, G)
        assert info["ranges"] >= 8 and info["ctas"] > 132, info
