"""Training a convolution layer on the device: pcnn_conv_plan_set_params (a plan refreshed from device memory computes what a
fresh plan computes, in stream order), pcnn_conv_bias_act_bwd (sigmoid derivative and bias gradient, bit-exact against a numpy
float32 replay and float64 sums) and ConvLayer (one step against float64 references, and a device training loop bit-identical
to a loop that re-creates its plans from host parameters every step)."""
import numpy as np
import pytest
import torch

import conv_ref as CR
import conv_ref_strided as CS

pytestmark = pytest.mark.gpu

NAN_BF16 = 0x7FC0

# N, H, W, C, K, R, S, stride: row-Toeplitz shapes (V = Toeplitz alignment variants)
NARROW = [
    (64, 28, 28, 1, 6, 5, 5, 1),        # LeNet c1, K = 6
    (3, 28, 28, 1, 6, 5, 5, 2),         # K = 6 at stride 2
    (2, 40, 60, 3, 16, 5, 5, 1),        # V = 2
    (2, 40, 60, 3, 8, 5, 5, 2),         # V = 2 at stride 2
    (2, 64, 40, 3, 64, 3, 3, 1),        # config-5-like, V = 2
    (2, 40, 60, 1, 64, 3, 5, 1),        # V = 2, C = 1
]
# N, H, W, C, K, R, S, stride, pad_h, pad_w: wide shapes
WIDE = [
    (2, 14, 14, 64, 64, 3, 3, 1, 0, 0),
    (2, 14, 14, 64, 64, 3, 3, 1, 1, 1),     # "same"
    (2, 13, 11, 40, 24, 5, 5, 1, 2, 2),     # K = 24, not a multiple of 16
    (2, 17, 15, 64, 40, 3, 3, 2, 1, 1),     # stride 2, K = 40
    (2, 12, 13, 320, 64, 3, 3, 1, 0, 0),    # C = 320
    (2, 12, 13, 320, 64, 3, 3, 1, 2, 2),    # C = 320, "full" padding
]


def nid(c):
    return "x".join(map(str, c[:7])) + f"-s{c[7]}"


def wid(c):
    return nid(c) + f"-pad{c[8]}{c[9]}"


def special_filters(rng, K, R, S, C):
    """random filters with, spread over the first filters: +-0, fp32 subnormals, exact bf16 ties (to even, both directions),
    finite values that round to +-Inf in bf16, and +-Inf"""
    f = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
    flat = f.reshape(-1)
    special = np.array([0.0, -0.0, 1e-40, -3e-39, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), 0.5 + 2.0 ** -9,
                        3.4e38, -3.39e38, np.inf, -np.inf], np.float32)
    idx = rng.choice(flat.size, special.size, replace=False)
    flat[idx] = special
    return f


def narrow_x(pkg, rng, N, H, W, C):
    pitch = (W * C + 7) // 8 * 8
    x = np.zeros((N * H, pitch), np.uint16)
    x[:, :W * C] = pkg.f32_to_bf16_bits(rng.uniform(0, 1, (N * H, W * C)).astype(np.float32))
    return x


def make_plan(pkg, eng, case, f, b, act=0):
    if len(case) == 8:
        N, H, W, C, K, R, S, st = case
        return pkg.ConvPlan(eng, N, H, W, C, K, R, S, f, b, act=act, stride=st)
    N, H, W, C, K, R, S, st, ph, pw = case
    return pkg.WideConvPlan(eng, N, H, W, C, K, R, S, f, b, act=act, stride=st, padding=(ph, pw))


def make_x(pkg, rng, case):
    N, H, W, C = case[:4]
    if len(case) == 8:
        return narrow_x(pkg, rng, N, H, W, C)
    return pkg.f32_to_bf16_bits(rng.uniform(0, 1, (N, H, W, C)).astype(np.float32))


def fwd(eng, plan, xd):
    y = eng.to_device(np.full(plan.out_shape, NAN_BF16, np.uint16))
    plan.fwd(xd, y)
    eng.sync()
    return y.to_host()


def fresh_fwd(pkg, eng, case, f, b, xd, act=0):
    plan = make_plan(pkg, eng, case, f, b, act)
    y = fwd(eng, plan, xd)
    plan.close()
    return y


# ------------------------------------------------------------------------------------------------ 1. refresh = fresh plan
@pytest.mark.parametrize("case", NARROW + WIDE, ids=[nid(c) for c in NARROW] + [wid(c) for c in WIDE])
def test_refresh_equals_fresh_plan(eng, pkg, case):
    K, R, S, C = case[4], case[5], case[6], case[3]
    rng = np.random.default_rng(sum(case))
    f0 = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
    b0 = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    f1 = special_filters(rng, K, R, S, C)
    b1 = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    xd = eng.to_device(make_x(pkg, rng, case))
    for act in (0, 1):
        plan = make_plan(pkg, eng, case, f0, b0, act)
        plan.set_params(eng.to_device(f1), eng.to_device(b1))
        got = fwd(eng, plan, xd)
        plan.close()
        want = fresh_fwd(pkg, eng, case, f1, b1, xd, act)
        assert np.array_equal(got, want), (act, int(np.sum(got != want)))
    # finite filters only: the refreshed plan computes finite outputs, so the test above compared real values
    fin = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
    plan = make_plan(pkg, eng, case, f0, None)
    plan.set_params(eng.to_device(fin))
    got = fwd(eng, plan, xd)
    plan.close()
    assert np.isfinite(pkg.bf16_bits_to_f32(got)).all()
    assert np.array_equal(got, fresh_fwd(pkg, eng, case, fin, None, xd))


@pytest.mark.parametrize("case", [NARROW[0], NARROW[2], WIDE[1], WIDE[2]], ids=[nid(NARROW[0]), nid(NARROW[2]), wid(WIDE[1]), wid(WIDE[2])])
def test_refresh_nan_filter(eng, pkg, case):
    """a NaN tap in filter k makes every output of channel k NaN (NaN * 0 is NaN) and no other, refreshed or fresh"""
    K, R, S, C = case[4], case[5], case[6], case[3]
    rng = np.random.default_rng(7)
    f0 = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
    f1 = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
    k = K - 1
    f1[k, R // 2, S - 1, C - 1] = np.nan
    xd = eng.to_device(make_x(pkg, rng, case))
    plan = make_plan(pkg, eng, case, f0, None)
    plan.set_params(eng.to_device(f1))
    got = pkg.bf16_bits_to_f32(fwd(eng, plan, xd))
    plan.close()
    want = pkg.bf16_bits_to_f32(fresh_fwd(pkg, eng, case, f1, None, xd))
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.isnan(got[..., k]).all() and np.isfinite(got[..., :k]).all()


# ------------------------------------------------------------------------------------------------ 2. stream order
@pytest.mark.parametrize("case", [NARROW[0], NARROW[4], WIDE[1]], ids=[nid(NARROW[0]), nid(NARROW[4]), wid(WIDE[1])])
def test_refresh_in_stream_order(eng, pkg, case):
    K, R, S, C = case[4], case[5], case[6], case[3]
    rng = np.random.default_rng(11)
    f0, f1 = (rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32) for _ in range(2))
    b0, b1, b2 = (rng.uniform(-0.5, 0.5, K).astype(np.float32) for _ in range(3))
    xd = eng.to_device(make_x(pkg, rng, case))
    f0d, f1d, b0d, b1d, b2d = (eng.to_device(a) for a in (f0, f1, b0, b1, b2))
    plan = make_plan(pkg, eng, case, f0, b0, act=1)
    ys = [eng.to_device(np.full(plan.out_shape, NAN_BF16, np.uint16)) for _ in range(4)]
    plan.fwd(xd, ys[0])                      # no synchronisation between any of these
    plan.set_params(f1d, b1d)
    plan.fwd(xd, ys[1])
    plan.set_params(f0d, b0d)
    plan.fwd(xd, ys[2])
    plan.set_params(None, b2d)               # bias only: the filters stay f0
    plan.fwd(xd, ys[3])
    eng.sync()
    got = [y.to_host() for y in ys]
    plan.close()
    want0 = fresh_fwd(pkg, eng, case, f0, b0, xd, act=1)
    assert np.array_equal(got[0], want0)
    assert np.array_equal(got[1], fresh_fwd(pkg, eng, case, f1, b1, xd, act=1))
    assert np.array_equal(got[2], want0)
    assert np.array_equal(got[3], fresh_fwd(pkg, eng, case, f0, b2, xd, act=1))


@pytest.mark.parametrize("case", [NARROW[0], WIDE[0]], ids=[nid(NARROW[0]), wid(WIDE[0])])
def test_refresh_refusals(eng, pkg, case):
    K, R, S, C = case[4], case[5], case[6], case[3]
    f = np.zeros((K, R, S, C), np.float32)
    plan = make_plan(pkg, eng, case, f, None)
    with pytest.raises(pkg.PcnnError, match="created without one"):
        plan.set_params(eng.to_device(f), eng.to_device(np.zeros(K, np.float32)))
    with pytest.raises(pkg.PcnnError, match="both NULL"):
        plan.set_params(None, None)
    plan.close()


# ------------------------------------------------------------------------------------------------ 3. pcnn_conv_bias_act_bwd
BA_THREADS, BA_ITERS = 256, 8


def n_acc(pixels, K):
    """longest chain of fp32 additions behind one db[k]: BA_ITERS pixels per thread, then the pixel lanes of a CTA in order, then
    pcnn_conv_wgrad_reduce_slots (8 strided chains over the CTA slots and a 3-level tree)"""
    lanes = BA_THREADS // (K // 8 if K % 8 == 0 else K)
    ctas = -(-pixels // (BA_ITERS * lanes))
    return BA_ITERS + lanes + -(-ctas // 8) + 3


def dpre_replay(pkg, y_bits, dy_bits):
    """numpy float32 replay of dpre = bf16_rn(dy * (y * (1 - y))): each float32 operation rounds to nearest, no contraction"""
    yf, gf = pkg.bf16_bits_to_f32(y_bits), pkg.bf16_bits_to_f32(dy_bits)
    return pkg.f32_to_bf16_bits(gf * (yf * (np.float32(1.0) - yf)))


def random_operands(pkg, rng, pixels, K):
    y = pkg.f32_to_bf16_bits(rng.uniform(0, 1, (pixels, K)).astype(np.float32))
    dy = pkg.f32_to_bf16_bits(rng.standard_normal((pixels, K)).astype(np.float32))
    return y, dy


def run_bias_act(eng, y, dy, act, with_db=True, in_place=False, tail=64):
    """dpre in a NaN-prefilled buffer `tail` elements longer than pixels * K; returns (dpre with tail, db, dy after)"""
    pixels, K = dy.shape
    yd = eng.to_device(y) if y is not None else None
    dyd = eng.to_device(dy)
    db = eng.to_device(np.full(K, np.nan, np.float32)) if with_db else None
    if in_place:
        dpre = dyd
    elif act:
        dpre = eng.to_device(np.full(pixels * K + tail, NAN_BF16, np.uint16))
    else:
        dpre = None
    eng.conv_bias_act_bwd(yd, dyd, dpre, db, pixels, K, act)
    eng.sync()
    return (dpre.to_host() if dpre is not None else None), (db.to_host() if with_db else None), dyd.to_host()


KS = [1, 6, 8, 16, 64, 120, 256]
PIXELS = [1, 7, 1001]
GRID = [(K, p) for K in KS for p in PIXELS] + [(64, 128 * 56 * 56)]


@pytest.mark.parametrize("K,pixels", GRID, ids=[f"K{K}-px{p}" for K, p in GRID])
def test_bias_act_random(eng, pkg, K, pixels):
    """dpre bit-identical to the float32 replay; db within 2 * n_acc * 2^-24 * sum |dpre| of the float64 sum of the same bf16
    values (fp32 summation model: each of the n_acc additions in a chain adds at most 2^-24 of the partial sum it forms, and
    every partial is bounded by sum |dpre|); NaN-prefilled dpre fully written, its tail untouched; in place = out of place;
    reruns bit-identical; db = NULL leaves dpre as it was"""
    rng = np.random.default_rng(K * 7919 + pixels)
    y, dy = random_operands(pkg, rng, pixels, K)
    n = pixels * K
    dpre, db, dy_after = run_bias_act(eng, y, dy, 1)
    want = dpre_replay(pkg, y, dy)
    assert np.array_equal(dpre[:n].reshape(pixels, K), want)
    assert np.all(dpre[n:] == NAN_BF16)
    assert np.array_equal(dy_after, dy)
    d64 = pkg.bf16_bits_to_f32(want).astype(np.float64)
    ref = d64.sum(axis=0)
    bound = 2 * n_acc(pixels, K) * 2.0 ** -24 * np.abs(d64).sum(axis=0)
    err = np.abs(db.astype(np.float64) - ref)
    assert np.all(err <= bound), (float(err.max()), float(bound.max()))
    ratio = float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1), 0)))
    print(f"K={K} pixels={pixels}: n_acc {n_acc(pixels, K)}, worst db error / bound {ratio:.3g}")
    _, db_ip, dy_ip = run_bias_act(eng, y, dy, 1, in_place=True)
    assert np.array_equal(dy_ip, want) and np.array_equal(db_ip, db)
    dpre2, db2, _ = run_bias_act(eng, y, dy, 1)
    assert np.array_equal(dpre2, dpre) and np.array_equal(db2, db)
    dpre3, _, _ = run_bias_act(eng, y, dy, 1, with_db=False)
    assert np.array_equal(dpre3, dpre)
    # act 0: db over dy, nothing written
    _, db0, dy0 = run_bias_act(eng, None, dy, 0)
    g64 = pkg.bf16_bits_to_f32(dy).astype(np.float64)
    assert np.array_equal(dy0, dy)
    assert np.all(np.abs(db0 - g64.sum(axis=0)) <= 2 * n_acc(pixels, K) * 2.0 ** -24 * np.abs(g64).sum(axis=0))


@pytest.mark.parametrize("K,pixels", GRID, ids=[f"K{K}-px{p}" for K, p in GRID])
def test_bias_act_integer_exact(eng, pkg, K, pixels):
    """dy in {-1, 0, 1}, y in {0, 1/2, 1}: y (1 - y) dy in {0, +-1/4} is exact, and so is every partial sum: db is bit-identical
    to the float64 sum, at act 1 and (over dy) at act 0"""
    rng = np.random.default_rng(K + pixels)
    y = pkg.f32_to_bf16_bits(rng.choice(np.array([0.0, 0.5, 1.0], np.float32), (pixels, K)))
    dy = pkg.f32_to_bf16_bits(rng.integers(-1, 2, (pixels, K)).astype(np.float32))
    dpre, db, _ = run_bias_act(eng, y, dy, 1)
    want = dpre_replay(pkg, y, dy)
    assert np.array_equal(dpre[:pixels * K].reshape(pixels, K), want)
    assert np.array_equal(db.astype(np.float64), pkg.bf16_bits_to_f32(want).astype(np.float64).sum(axis=0))
    _, db0, _ = run_bias_act(eng, None, dy, 0)
    assert np.array_equal(db0.astype(np.float64), pkg.bf16_bits_to_f32(dy).astype(np.float64).sum(axis=0))


def test_bias_act_refusals(eng, pkg):
    K, pixels = 16, 64
    y, dy, dpre = (eng.array((pixels + 8, K), np.uint16) for _ in range(3))
    db = eng.array(K + 8)
    call = eng.conv_bias_act_bwd
    cases = [
        (lambda: call(y, dy, dpre, db, pixels, 0, 1), "1 <= K <= 256"),
        (lambda: call(y, dy, dpre, db, pixels, 257, 1), "1 <= K <= 256"),
        (lambda: call(y, dy, dpre, db, 0, K, 1), "at least one pixel"),
        (lambda: call(y, dy, dpre, db, pixels, K, 2), "act 2"),
        (lambda: call(None, dy, dpre, db, pixels, K, 1), "needs y"),
        (lambda: call(y, dy, None, db, pixels, K, 1), "needs y"),
        (lambda: call(None, dy, dpre, db, pixels, K, 0), "act 0 writes no dpre"),
        (lambda: call(None, dy, None, None, pixels, K, 0), "act 0 writes no dpre"),
        (lambda: call(y, None, dpre, db, pixels, K, 1), "NULL context or dy"),
        (lambda: call(y, dy.ptr + 2, dpre, db, pixels, K, 1), "16-byte aligned"),
        (lambda: call(y, dy, dpre.ptr + 8, db, pixels, K, 1), "16-byte aligned"),
        (lambda: call(y, dy, dpre, db.ptr + 4, pixels, K, 1), "16-byte aligned"),
        (lambda: call(y, dy, dy.ptr + 16, db, pixels, K, 1), "overlapping"),
        (lambda: call(y, dy, y, db, pixels, K, 1), "overlapping"),
        (lambda: call(y, dy, dpre, dy, pixels, K, 1), "overlapping"),
        (lambda: call(y, dy, dpre, y, pixels, K, 1), "overlapping"),
    ]
    for fn, msg in cases:
        with pytest.raises(pkg.PcnnError, match=msg):
            fn()
    call(y, dy, dy, db, pixels, K, 1)        # in place is allowed
    eng.sync()


# ------------------------------------------------------------------------------------------------ 4. one layer step vs float64
def _int_layer_operands(rng, N, H, W, C, K, R, S, P, Q):
    x = rng.integers(0, 4, (N, H, W, C)).astype(np.float32)
    dens = min(0.5, 48.0 / max(R * S * C, K * R * S))
    f = ((rng.random((K, R, S, C)) < dens) * rng.choice(np.array([-1, 1], np.float32), (K, R, S, C))).astype(np.float32)
    b = rng.integers(-2, 3, K).astype(np.float32)
    dy = rng.integers(-1, 2, (N, P, Q, K)).astype(np.float32)
    return x, f, b, dy


LAYERS = [  # N, H, W, C, K, R, S, stride, pad: one narrow (row-Toeplitz) and one wide layer
    (8, 28, 28, 1, 8, 5, 5, 1, 0),
    (4, 24, 24, 8, 16, 3, 3, 1, 1),
]


def _layer_step(eng, pkg, case, x, f, b, dy_bits, act):
    N, H, W, C, K, R, S, st, pad = case
    layer = pkg.ConvLayer(eng, N, H, W, C, K, R, S, f, b, act=act, stride=st, padding=(pad, pad))
    pitch = layer.row_pitch
    xl = np.zeros((N * H, pitch), np.uint16)
    xl[:, :W * C] = pkg.f32_to_bf16_bits(x).reshape(N * H, W * C)
    xd = eng.to_device(xl)
    y = eng.to_device(np.full(layer.out_shape, NAN_BF16, np.uint16))
    dyd = eng.to_device(dy_bits)
    dx = eng.to_device(np.full((N * H, pitch), NAN_BF16, np.uint16))
    layer.forward(xd, y)
    layer.backward(y, dyd, dx)
    eng.sync()
    out = dict(y=y.to_host(), dpre=dyd.to_host(), dw=layer.dw.to_host(), db=layer.db.to_host(),
               dx=dx.to_host()[:, :W * C].reshape(N, H, W, C), family=layer.family)
    layer.close()
    return out


def _refs(pkg, case, x, f, dpre):
    N, H, W, C, K, R, S, st, pad = case
    xp = np.pad(x.astype(np.float64), ((0, 0), (pad, pad), (pad, pad), (0, 0)))
    dw = CS.conv_wgrad_f64(xp, dpre, R, S, st)
    dx = CS.conv_dgrad_f64(dpre, f.astype(np.float64), H + 2 * pad, W + 2 * pad, st)[:, pad:pad + H, pad:pad + W, :]
    # sums of |terms|: the scale of the fp32 accumulation error
    dw_abs = CS.conv_wgrad_f64(np.abs(xp), np.abs(dpre), R, S, st)
    dx_abs = CS.conv_dgrad_f64(np.abs(dpre), np.abs(f.astype(np.float64)), H + 2 * pad, W + 2 * pad, st)[:, pad:pad + H, pad:pad + W, :]
    return dw, dx, dw_abs, dx_abs


@pytest.mark.parametrize("case", LAYERS, ids=["narrow", "wide"])
def test_layer_step_integer_exact(eng, pkg, case):
    """act 0 with bias, integer operands: dw, db and dx are exact"""
    N, H, W, C, K, R, S, st, pad = case
    P, Q = (H + 2 * pad - R) // st + 1, (W + 2 * pad - S) // st + 1
    rng = np.random.default_rng(3)
    x, f, b, dy = _int_layer_operands(rng, N, H, W, C, K, R, S, P, Q)
    out = _layer_step(eng, pkg, case, x, f, b, pkg.f32_to_bf16_bits(dy), act=0)
    assert out["family"] == ("narrow" if pad == 0 else "wide")
    xp = np.pad(x.astype(np.float64), ((0, 0), (pad, pad), (pad, pad), (0, 0)))
    assert np.array_equal(pkg.bf16_bits_to_f32(out["y"]), CR.conv_fwd_f64(xp, f, b, st).astype(np.float32))
    assert np.array_equal(out["dpre"], pkg.f32_to_bf16_bits(dy))          # act 0: dy is not rewritten
    dw, dx, _, _ = _refs(pkg, case, x, f, dy.astype(np.float64))
    assert np.array_equal(out["dw"].astype(np.float64), dw)
    assert np.array_equal(out["db"].astype(np.float64), dy.astype(np.float64).sum(axis=(0, 1, 2)))
    assert np.array_equal(pkg.bf16_bits_to_f32(out["dx"]).astype(np.float64), dx)


@pytest.mark.parametrize("case", LAYERS, ids=["narrow", "wide"])
def test_layer_step_sigmoid_random(eng, pkg, case):
    """act 1 with bias, random operands.  dpre (dy rewritten in place) is the float32 replay on the layer's own y; dw, db and dx
    against float64 on that dpre and the bf16 operands: fp32 accumulation within 2 n 2^-24 sum |terms| (n terms per output),
    dx also within its bf16 rounding (2^-8 relative)"""
    N, H, W, C, K, R, S, st, pad = case
    P, Q = (H + 2 * pad - R) // st + 1, (W + 2 * pad - S) // st + 1
    rng = np.random.default_rng(5)
    x = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(0, 1, (N, H, W, C)).astype(np.float32)))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    dy = pkg.f32_to_bf16_bits(rng.standard_normal((N, P, Q, K)).astype(np.float32))
    out = _layer_step(eng, pkg, case, x, f, b, dy, act=1)
    assert np.array_equal(out["dpre"], dpre_replay(pkg, out["y"], dy))
    dpre = pkg.bf16_bits_to_f32(out["dpre"]).astype(np.float64)
    dw, dx, dw_abs, dx_abs = _refs(pkg, case, x, f, dpre)
    npix = N * P * Q
    assert np.all(np.abs(out["dw"] - dw) <= 2 * npix * 2.0 ** -24 * dw_abs + 1e-30)
    db_ref = dpre.sum(axis=(0, 1, 2))
    assert np.all(np.abs(out["db"] - db_ref) <= 2 * npix * 2.0 ** -24 * np.abs(dpre).sum(axis=(0, 1, 2)))
    got_dx = pkg.bf16_bits_to_f32(out["dx"]).astype(np.float64)
    assert np.all(np.abs(got_dx - dx) <= 2.0 ** -8 * np.abs(dx) + 2 * K * R * S * 2.0 ** -24 * dx_abs + 1e-30)


# ------------------------------------------------------------------------------------------------ 5. device loop = host loop
LR = 2.0 ** -20


class TwoLayers:
    """28x28x1 -> 8@5x5 sigmoid + bias (row-Toeplitz, no dx) -> 16@3x3 padding 1 + bias (wide), loss 1/2 |y2 - t|^2"""

    def __init__(self, eng, pkg, B, params):
        self.eng, self.pkg, self.B = eng, pkg, B
        f1, b1, f2, b2 = params
        self.l1 = pkg.ConvLayer(eng, B, 28, 28, 1, 8, 5, 5, f1, b1, act=1)
        self.l2 = pkg.ConvLayer(eng, B, 24, 24, 8, 16, 3, 3, f2, b2, act=0, padding=(1, 1))
        assert (self.l1.family, self.l2.family) == ("narrow", "wide")
        dev = torch.device("cuda", 0)
        self.y1 = torch.empty((B, 24, 24, 8), dtype=torch.int16, device=dev)
        self.dy1 = torch.empty_like(self.y1)
        self.y2 = torch.empty((B, 24, 24, 16), dtype=torch.int16, device=dev)
        self.dy2 = torch.empty_like(self.y2)

    def step(self, xd, t, refresh):
        """one SGD step; returns the loss of the forward it starts with"""
        self.l1.forward(xd, self.y1)
        self.l2.forward(self.y1, self.y2)
        self.eng.sync()
        e = self.y2.view(torch.bfloat16).float() - t
        self.dy2.view(torch.bfloat16).copy_(e.to(torch.bfloat16))
        loss = 0.5 * float((e.double() ** 2).sum())
        torch.cuda.synchronize()
        self.l2.backward(self.y2, self.dy2, self.dy1)
        self.l1.backward(self.y1, self.dy1, None)
        refresh(self.l1)
        refresh(self.l2)
        self.eng.sync()
        return loss

    def params(self):
        return [a for layer in (self.l1, self.l2) for a in layer.params()]

    def grads(self):
        return [a.to_host() for layer in (self.l1, self.l2) for a in (layer.dw, layer.db)]

    def close(self):
        self.l1.close()
        self.l2.close()


def _host_refresh(pkg, eng, layer, lr):
    """the same update on the device masters, then a new plan built from their host copy (the old plan destroyed)"""
    n = int(np.prod(layer.shape[3:]))
    eng.apply_grad_scaled(layer.filt, layer.dw, n, -lr)
    eng.apply_grad_scaled(layer.bias, layer.db, layer.shape[4], -lr)
    f, b = layer.params()
    N, H, W, C, K, R, S = layer.shape
    layer.plan.close()
    if layer.family == "narrow":
        layer.plan = pkg.ConvPlan(eng, N, H, W, C, K, R, S, f, b, act=layer.act, stride=layer.stride)
    else:
        layer.plan = pkg.WideConvPlan(eng, N, H, W, C, K, R, S, f, b, act=layer.act, stride=layer.stride, padding=layer.padding)


def test_device_loop_equals_host_loop(eng, pkg, golden):
    B = 64
    rng = np.random.default_rng(2024)
    params = [rng.uniform(-0.2, 0.2, (8, 5, 5, 1)).astype(np.float32), rng.uniform(-0.2, 0.2, 8).astype(np.float32),
              rng.uniform(-0.1, 0.1, (16, 3, 3, 8)).astype(np.float32), rng.uniform(-0.1, 0.1, 16).astype(np.float32)]
    imgs = golden["train_u8"][:B].reshape(B, 28, 28).astype(np.float32) / 255.0
    xl = np.zeros((B * 28, 32), np.uint16)
    xl[:, :28] = pkg.f32_to_bf16_bits(imgs).reshape(B * 28, 28)
    xd = eng.to_device(xl)
    t = torch.from_numpy(rng.uniform(0, 1, (B, 24, 24, 16)).astype(np.float32)).cuda()
    dev_net, host_net = TwoLayers(eng, pkg, B, params), TwoLayers(eng, pkg, B, params)
    losses = []
    for it in range(20):
        before = dev_net.params()
        losses.append(dev_net.step(xd, t, lambda layer: layer.sgd(LR)))
        if it < 5:
            host_net.step(xd, t, lambda layer: _host_refresh(pkg, eng, layer, LR))
            after_dev, after_host = dev_net.params(), host_net.params()
            for a, h in zip(after_dev, after_host):
                assert np.array_equal(a.view(np.uint32), h.view(np.uint32)), it
            # w <- w + (-lr) * dw: one float32 multiply, then one float32 add
            for w0, g, w1 in zip(before, dev_net.grads(), after_dev):
                assert np.array_equal((w0 + np.float32(-LR) * g).view(np.uint32), w1.view(np.uint32)), it
    dev_net.close()
    host_net.close()
    print("loss over 20 steps:", " ".join(f"{v:.4g}" for v in losses))
    assert losses[-1] < losses[0]
