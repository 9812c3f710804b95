"""SiLU, hard-swish and ReLU6 after batch normalization, on the host: the replayable exponential E within its stated bound over
the finite fp32 inputs, the float64 references of bnact_ref.py pinned to torch's CPU float64 activations and autograd (special
values and knees included), the whole BN + r + act block against torch autograd in the layer's backward order, the two shortcuts
the backward must not take (a ReLU6 mask from the bf16 y, a pre-activation without r), and the float32 replays within float32
rounding of float64."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import bnact_ref as AR

TF = {AR.SILU: F.silu, AR.HARDSWISH: F.hardswish, AR.RELU6: F.relu6}
SPECIAL = [np.nan, -np.inf, np.inf, -0.0, 0.0, -3.0, 3.0, 6.0, -6.0, np.nextafter(-3.0, 0), np.nextafter(-3.0, -4),
           np.nextafter(3.0, 0), np.nextafter(3.0, 4), np.nextafter(6.0, 0), np.nextafter(6.0, 7), 5.99, 5.985, -1.28, -1.5, 1e-30,
           -1e-30, 88.72, 88.73, -88.72, -88.73, -103.9, -104.0, 87.0, -87.0, 1e30, -1e30, 3.0e38, -3.0e38]


def padded(v, n=64):
    """torch runs the body of a tensor through its vectorised loop: pad to a multiple of 64 elements so every value takes it"""
    v = np.asarray(v, np.float64)
    return np.concatenate([v, np.zeros(-v.size % n)])


def close(a, b, tol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    nan = np.isnan(b)
    same_inf = np.isinf(b) & (a == b)
    ok = np.isnan(a) == nan
    fin = ~nan & ~np.isinf(b)
    ok &= np.where(np.isinf(b), same_inf, True)
    with np.errstate(invalid="ignore"):
        ok &= np.where(fin, np.abs(a - b) <= tol * np.maximum(1.0, np.abs(b)), True)
    return bool(ok.all())


# ------------------------------------------------------------------------------------------------ E
def ulp_error(x):
    """|E(x) - exp(x)| in units of the fp32 spacing at exp(x) (2^-149 for subnormal results); exact +Inf and +0 past the
    thresholds"""
    got = AR.exp_f32(x).astype(np.float64)
    with np.errstate(over="ignore"):
        ref = np.exp(x.astype(np.float64))
    ulp = np.maximum(np.abs(np.spacing(np.minimum(ref, 3.4e38).astype(np.float32))).astype(np.float64), 2.0 ** -149)
    with np.errstate(invalid="ignore"):
        return np.where(np.isinf(got) & (ref > 3.4028235677973366e38), 0.0, np.abs(got - ref) / ulp)


def test_exp_sweep_within_the_stated_bound():
    """every 97th bit pattern of both signs over the finite range, the thresholds and their neighbours, subnormal results, +-0,
    +-Inf and NaN: within E_MAX_ULP of float64 exp, +Inf above the overflow threshold, +0 below the underflow one"""
    pos = np.arange(0, 0x7F800000, 97, dtype=np.uint32)
    x = np.concatenate([pos, pos | np.uint32(0x80000000)]).view(np.float32)
    edges = np.array([0x42B17216, 0x42B17217, 0x42B17218, 0xC2CFF1B3, 0xC2CFF1B4, 0xC2CFF1B5, 0xC2AEAC4F, 0xC2AEAC50, 0xC2AEAC51],
                     np.uint32).view(np.float32)
    sub = np.linspace(-103.97, -87.33, 200001).astype(np.float32)           # results in the subnormal range
    x = np.concatenate([x, edges, sub, np.float32([0.0, -0.0, 1.0, -1.0])])
    e = ulp_error(x)
    worst = float(e.max())
    print(f"E: max error {worst:.4f} ulp over {x.size} inputs at x = {x[e.argmax()]!r}; correctly rounded {float((e <= 0.5).mean()):.4f}")
    assert worst <= AR.E_MAX_ULP
    assert worst > AR.E_MAX_ULP - 0.01                                      # the bound is the measured maximum, not slack
    assert np.all(AR.exp_f32(x[x > AR.E_HI]) == np.inf) and np.all(AR.exp_f32(x[x < AR.E_LO]) == 0)
    assert np.all(AR.exp_f32(x[(x <= AR.E_HI) & (x >= AR.E_LO)]) > 0)
    assert not np.isinf(AR.exp_f32(AR.E_HI)) and AR.exp_f32(AR.E_LO) == np.float32(2.0 ** -149)
    sp = AR.exp_f32(np.float32([np.inf, -np.inf, np.nan, 0.0, -0.0]))
    assert sp[0] == np.inf and sp[1] == 0 and not np.signbit(sp[1]) and np.isnan(sp[2]) and sp[3] == 1 and sp[4] == 1


# ------------------------------------------------------------------------------------------------ float64 references vs torch
@pytest.mark.parametrize("code", AR.CODES, ids=[AR.NAMES[c] for c in AR.CODES])
def test_f64_references_equal_torch(code):
    """act_f64 and dact_f64 equal torch's float64 activation and its autograd within 1e-12, NaN where torch gives NaN, the sign
    of a zero where torch keeps one, at the knees, the special values and random values"""
    rng = np.random.default_rng(code)
    v = padded(np.concatenate([SPECIAL, rng.standard_normal(500) * 4, rng.uniform(-8, 8, 500)]))
    t = padded(np.concatenate([np.full(len(SPECIAL), 2.0), rng.standard_normal(1000)]))
    vt = torch.from_numpy(v).requires_grad_(True)
    y = TF[code](vt)
    y.backward(torch.from_numpy(t))
    assert close(AR.act_f64(v, code), y.detach().numpy()) and close(AR.dact_f64(v, t, code), vt.grad.numpy())
    zero = (y.detach().numpy() == 0)
    assert np.array_equal(np.signbit(AR.act_f64(v, code)[zero]), np.signbit(y.detach().numpy()[zero]))


# ------------------------------------------------------------------------------------------------ the block
def torch_block(x, gamma, beta, r, dy, dy2, code, N, H, W):
    M, C = x.shape
    nchw = lambda a: torch.from_numpy(np.asarray(a, np.float64)).reshape(N, H, W, C).permute(0, 3, 1, 2)
    xt = nchw(x).requires_grad_(True)
    rt = None if r is None else nchw(r).requires_grad_(True)
    gt, bt = torch.from_numpy(gamma.astype(np.float64)).requires_grad_(True), torch.from_numpy(beta.astype(np.float64)).requires_grad_(True)
    v = F.batch_norm(xt, None, None, gt, bt, training=True, eps=1e-5)
    if rt is not None:
        v = v + rt
    y = TF[code](v)
    y.backward(nchw(np.asarray(dy, np.float64) + (0 if dy2 is None else np.asarray(dy2, np.float64))))
    back = lambda a: a.detach().permute(0, 2, 3, 1).reshape(M, C).numpy()
    return back(y), back(xt.grad), gt.grad.numpy(), bt.grad.numpy(), None if rt is None else back(rt.grad)


def block_operands(rng, M, C):
    x = rng.standard_normal((M, C)) * 2 + 1
    gamma, beta = rng.uniform(0.5, 3, C), rng.uniform(-2, 4, C)
    return x, gamma, beta, rng.standard_normal((M, C)) * 2, rng.standard_normal((M, C)), rng.standard_normal((M, C))


@pytest.mark.parametrize("code", AR.CODES, ids=[AR.NAMES[c] for c in AR.CODES])
@pytest.mark.parametrize("with_r,with_dy2", [(True, True), (True, False), (False, True), (False, False)])
def test_block_f64_equals_torch_autograd(code, with_r, with_dy2):
    """block_f64 (y, dx, dgamma, dbeta and dr = g) equals torch's autograd of batch_norm(...) + r followed by the activation"""
    N, H, W, C = 4, 5, 7, 16
    rng = np.random.default_rng(code * 7 + with_r * 2 + with_dy2)
    x, gamma, beta, r, dy, dy2 = block_operands(rng, N * H * W, C)
    r, dy2 = (r if with_r else None), (dy2 if with_dy2 else None)
    y, _, dx, dg, db, g = AR.block_f64(x, gamma, beta, r, dy, dy2, code)
    ty, tdx, tdg, tdb, tdr = torch_block(x, gamma, beta, r, dy, dy2, code, N, H, W)
    for a, b in ((y, ty), (dx, tdx), (dg, tdg), (db, tdb)) + (((g, tdr),) if with_r else ()):
        assert np.allclose(a, b, rtol=1e-10, atol=1e-12)


def test_shortcuts_the_backward_must_not_take(pkg):
    """ReLU6's mask taken from the bf16 y zeroes the gradient of every v in (5.984, 6), which bf16 rounds to y = 6, where torch
    passes it; a pre-activation recomputed without r gives a different dx wherever r moves v across a knee"""
    N, H, W, C = 4, 5, 7, 16
    M = N * H * W
    rng = np.random.default_rng(5)
    x, gamma, beta, r, dy, _ = block_operands(rng, M, C)
    band = np.linspace(5.9845, 5.9999, 50)
    assert np.all(np.float64(np.float32(band).astype(np.float32)) < 6)
    yb = pkg.f32_to_bf16_bits(band.astype(np.float32))
    assert np.all(pkg.bf16_bits_to_f32(yb) == 6)                          # bf16 rounds every one of them to 6
    from_y = AR.dact_f64(pkg.bf16_bits_to_f32(yb).astype(np.float64), np.ones(50), AR.RELU6)
    assert np.all(from_y == 0) and np.all(AR.dact_f64(band, np.ones(50), AR.RELU6) == 1)
    tv = torch.from_numpy(band).requires_grad_(True)
    F.relu6(tv).backward(torch.ones(50, dtype=torch.float64))
    assert np.all(tv.grad.numpy() == 1)                                   # torch passes them
    for code in AR.CODES:
        _, _, dx, _, _, _ = AR.block_f64(x, gamma, beta, r, dy, None, code)
        _, _, dx0, _, _, _ = AR.block_f64(x, gamma, beta, None, dy, None, code)
        assert not np.allclose(dx0, dx, rtol=1e-3, atol=1e-3), code
        _, tdx, _, _, _ = torch_block(x, gamma, beta, r, dy, None, code, N, H, W)
        assert np.allclose(dx, tdx, rtol=1e-10, atol=1e-12)


# ------------------------------------------------------------------------------------------------ float32 replays
@pytest.mark.parametrize("code", AR.CODES, ids=[AR.NAMES[c] for c in AR.CODES])
def test_f32_replays_track_f64(pkg, code):
    """act32 within a few fp32 roundings of float64 (exactly at the specials); g within bf16 rounding of float64's
    dact(v) * t, with t rounded as the kernels round it"""
    rng = np.random.default_rng(40 + code)
    v = np.concatenate([np.float32(SPECIAL), (rng.standard_normal(20000) * 5).astype(np.float32),
                        rng.uniform(-100, 100, 2000).astype(np.float32)]).astype(np.float32)
    a32 = AR.act32(v, code).astype(np.float64)
    a64 = AR.act_f64(v.astype(np.float64), code)
    nan = np.isnan(a64)
    assert np.array_equal(np.isnan(a32), nan)
    fin = ~nan & np.isfinite(a64)
    assert np.all(a32[~nan & ~fin] == a64[~nan & ~fin])
    # SiLU: E's 1.3 ulp and 3 roundings, on a quotient whose conditioning is at most 1 + |v| e^-v / (1 + e^-v) <= 1 + |v|
    k = {AR.SILU: 6 * (1 + np.abs(v[fin])), AR.HARDSWISH: 4.0, AR.RELU6: 0.0}[code]
    over = (-v[fin] > AR.E_HI) if code == AR.SILU else np.zeros(fin.sum(), bool)
    if code == AR.HARDSWISH:                          # RN(v u) overflows for v > FLT_MAX / 6: +Inf, as torch's float32 hardswish
        big = v[fin].astype(np.float64) * 6 > np.finfo(np.float32).max
        assert np.all(a32[fin][big] == np.inf)
        fin &= ~(v.astype(np.float64) * 6 > np.finfo(np.float32).max)
        over = np.zeros(fin.sum(), bool)
    # SiLU below -88.72: E(-v) is +Inf and y is -0 where float64 has |v| e^v < 2^-119, as torch's float32 silu gives
    assert np.all((a32[fin][over] == 0) & np.signbit(a32[fin][over]) & (np.abs(a64[fin][over]) < 2.0 ** -119))
    a32f, a64f = a32[fin][~over], a64[fin][~over]
    k = k[~over] if code == AR.SILU else k
    vf = np.abs(v[fin][~over].astype(np.float64))
    # hard-swish: RN(v + 3) cancels near v = -3, an absolute |v| (|v| + 3) / 6 u
    slack = vf * (vf + 3) / 6 * 2.0 ** -23 if code == AR.HARDSWISH else 0.0
    assert np.all(np.abs(a32f - a64f) <= k * 2.0 ** -24 * np.abs(a64f) + slack + 2.0 ** -149)
    dyb = pkg.f32_to_bf16_bits(rng.standard_normal(v.size).astype(np.float32))
    g = pkg.bf16_bits_to_f32(AR.grad_bits(pkg, v, dyb, None, code)).astype(np.float64)
    g64 = AR.dact_f64(v.astype(np.float64), pkg.bf16_bits_to_f32(dyb).astype(np.float64), code)
    nan = np.isnan(g64)
    assert np.array_equal(np.isnan(g), nan)
    # d cancels where the derivative crosses 0 (SiLU at v = -1.278, hard-swish at -1.5): a few fp32 roundings of its terms, absolute
    t = np.abs(pkg.bf16_bits_to_f32(dyb).astype(np.float64))[~nan]
    with np.errstate(invalid="ignore"):
        slack = np.where(np.isfinite(v[~nan]), t * 2.0 ** -20 * (1 + np.abs(v[~nan].astype(np.float64))), 0.0)
    assert np.all(np.abs(g[~nan] - g64[~nan]) <= 2.0 ** -8 * np.abs(g64[~nan]) * (1 + 1e-4) + slack + 1e-38)
    # without dy2 a passed gradient keeps dy's bits
    passed = {AR.SILU: np.zeros(v.size, bool), AR.HARDSWISH: v >= 3, AR.RELU6: (v > 0) & (v < 6)}[code]
    assert np.array_equal(AR.grad_bits(pkg, v, dyb, None, code)[passed], dyb[passed])
