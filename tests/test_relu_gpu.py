"""ReLU (act 3, PCNN_ACT_RELU) in the device-trained layers: the forward epilogues of the row-Toeplitz, wide and linear plans bit
for bit against relu_ref.py on exact integer operands (with +-Inf and NaN biases), act 3 against act 0 on random operands,
pcnn_conv_bias_act_bwd at act 3 bit-exact with its refusals, one layer step of each family against float64, and a LeNet-style
classifier with ReLU layers trained on MNIST digits."""
import numpy as np
import pytest
import torch

import conv_ref as CR
import conv_ref_strided as CS
import linear_ref as LR
import relu_ref as RR
from example_nets import DEV, NAN_BF16, ReluNet, host, nan_buf, train

pytestmark = pytest.mark.gpu

TAIL = 64                      # elements past every output, prefilled with NaN: never written

# N, H, W, C, K, R, S, stride: row-Toeplitz shapes
NARROW = [
    (64, 28, 28, 1, 6, 5, 5, 1),        # LeNet c1, K = 6
    (3, 28, 28, 1, 6, 5, 5, 2),         # K = 6 at stride 2
    (2, 40, 60, 3, 16, 5, 5, 1),        # V = 2
]
# N, H, W, C, K, R, S, stride, pad: wide shapes
WIDE = [
    (2, 14, 14, 64, 64, 3, 3, 1, 0),    # unpadded
    (2, 14, 14, 64, 64, 3, 3, 1, 1),    # "same"
    (2, 17, 15, 64, 40, 3, 3, 2, 1),    # stride 2, pad 1
    (2, 12, 13, 320, 64, 3, 3, 1, 2),   # C = 320, "full"
]
# id, N, P, Q, C, O, row_pitch (0 = Q*C rounded up to 8), image_rows (0 = P)
LINEAR = [
    ("n200-o1", 200, 2, 3, 8, 1, 0, 0),
    ("lenet-fc2-o10", 128, 1, 1, 128, 10, 128, 1),
    ("fc-after-fc-o16", 300, 1, 1, 128, 16, 0, 0),
    ("n129-o256-qc80", 129, 2, 2, 40, 256, 0, 0),
    ("n100-qc130-pitched-fwdsplit", 100, 6, 5, 26, 10, 144, 8),
    ("head-7x7x256-n1024", 1024, 7, 7, 256, 256, 0, 0),
    ("head-1x1x2048-n4096", 4096, 1, 1, 2048, 256, 0, 0),
]
CONV = NARROW + WIDE


def cid(c):
    return "x".join(map(str, c[:7])) + f"-s{c[7]}" + (f"-pad{c[8]}" if len(c) == 9 else "")


def dev_bits(bits):
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).to(DEV)


def same_or_nan(got, want):
    """bf16 bits: identical where want is a number; NaN (any payload) where want is NaN"""
    nan, gnan = (want & 0x7FFF) > 0x7F80, (got & 0x7FFF) > 0x7F80
    return np.array_equal(gnan, nan) and np.array_equal(got[~nan], want[~nan])


# ------------------------------------------------------------------------------------------------ plans and their x layouts
def conv_geometry(case):
    N, H, W, C, K, R, S, st = case[:8]
    pad = case[8] if len(case) == 9 else 0
    return N, H, W, C, K, R, S, st, pad, (H + 2 * pad - R) // st + 1, (W + 2 * pad - S) // st + 1


def conv_plan(pkg, eng, case, f, b, act):
    N, H, W, C, K, R, S, st, pad, _, _ = conv_geometry(case)
    if len(case) == 8:
        return pkg.ConvPlan(eng, N, H, W, C, K, R, S, f, b, act=act, stride=st)
    return pkg.WideConvPlan(eng, N, H, W, C, K, R, S, f, b, act=act, stride=st, padding=(pad, pad))


def conv_x(pkg, x):
    """x [N][H][W][C] into [N * H][pitch] with NaN in the pad columns (never read)"""
    N, H, W, C = x.shape
    pitch = (W * C + 7) // 8 * 8
    buf = np.full((N * H, pitch), NAN_BF16, np.uint16)
    buf[:, :W * C] = pkg.f32_to_bf16_bits(x).reshape(N * H, W * C)
    return dev_bits(buf)


def linear_x(pkg, x, pitch, rows):
    N, P, Q, C = x.shape
    buf = np.full((N, rows, pitch), NAN_BF16, np.uint16)
    buf[:, :P, :Q * C] = pkg.f32_to_bf16_bits(x).reshape(N, P, Q * C)
    return dev_bits(buf)


def linear_layout(case):
    _, N, P, Q, C, O, pitch, rows = case
    return (pitch or (Q * C + 7) // 8 * 8), (rows or P)


def run_fwd(plan, xd, n_out):
    """y in a NaN-prefilled buffer TAIL elements longer than the output; returns all of it"""
    y = nan_buf(n_out + TAIL)
    torch.cuda.synchronize()
    plan.fwd(xd, y)
    plan.engine.sync()
    return host(y)


def special_bias(b):
    """channel 0 +Inf (y +Inf), channel 1 -Inf (y +0), the last channel NaN (y NaN)"""
    b = b.copy()
    b[0] = np.inf
    if b.size > 1:
        b[1] = -np.inf
    if b.size > 2:
        b[-1] = np.nan
    return b


# ------------------------------------------------------------------------------------------------ 1. forward, exact
@pytest.mark.parametrize("case", CONV, ids=[cid(c) for c in CONV])
def test_conv_forward_exact(eng, pkg, case):
    """x in -2..2, sparse +-1 filters, integer bias: every fp32 sum is exact and about half of them are negative.  y is
    bf16_rn(relu(v)) bit for bit, the special biases give +Inf, +0 and NaN, the tail stays NaN and a rerun gives the same bits"""
    N, H, W, C, K, R, S, st, pad, P, Q = conv_geometry(case)
    rng = np.random.default_rng(sum(case))
    x = rng.integers(-2, 3, (N, H, W, C)).astype(np.float32)
    dens = min(0.5, 48.0 / (R * S * C))
    f = ((rng.random((K, R, S, C)) < dens) * rng.choice(np.array([-1, 1], np.float32), (K, R, S, C))).astype(np.float32)
    b = special_bias(rng.integers(-2, 3, K).astype(np.float32))
    plan = conv_plan(pkg, eng, case, f, b, pkg.ACT_RELU)
    xd = conv_x(pkg, x)
    n = N * P * Q * K
    y = run_fwd(plan, xd, n)
    xp = np.pad(x.astype(np.float64), ((0, 0), (pad, pad), (pad, pad), (0, 0)))
    with np.errstate(invalid="ignore"):
        v = CR.conv_fwd_f64(xp, f, b, st)
    want = RR.fwd_bits(pkg, v).reshape(-1)
    assert same_or_nan(y[:n], want)
    yf = pkg.bf16_bits_to_f32(y[:n]).reshape(N, P, Q, K)
    assert np.all(yf[..., 0] == np.inf) and np.all(y[:n].reshape(N, P, Q, K)[..., 1] == 0) and np.isnan(yf[..., -1]).all()
    fin = v[..., 2:-1]
    neg = float((fin < 0).mean())
    assert 0.2 < neg < 0.8, neg
    assert not np.any(y[:n] == 0x8000)
    assert np.all(y[n:] == NAN_BF16)
    assert np.array_equal(run_fwd(plan, xd, n), y)
    plan.close()
    print(f"{cid(case)}: {neg:.2f} of the finite pre-activations negative")


@pytest.mark.parametrize("case", LINEAR, ids=[c[0] for c in LINEAR])
def test_linear_forward_exact(eng, pkg, case):
    """integer x, W, b in -3..3 (sums exact, about half negative), split and unsplit reductions: y bit for bit, special biases,
    NaN in x's pad never read, the tail untouched, reruns identical"""
    name, N, P, Q, C, O, _, _ = case
    pitch, rows = linear_layout(case)
    info = pkg.linear_info(N, P, Q, C, O, pitch, rows)
    rng = np.random.default_rng(N + 7 * O)
    x = rng.integers(-3, 4, (N, P, Q, C)).astype(np.float32)
    w = rng.integers(-3, 4, (O, P, Q, C)).astype(np.float32)
    b = special_bias(rng.integers(-8, 9, O).astype(np.float32))
    plan = pkg.LinearPlan(eng, N, P, Q, C, O, w, b, act=pkg.ACT_RELU, row_pitch=pitch, image_rows=rows)
    xd = linear_x(pkg, x, pitch, rows)
    n = N * O
    y = run_fwd(plan, xd, n)
    with np.errstate(invalid="ignore"):
        v = LR.fwd_f64(x, w, b)
    assert same_or_nan(y[:n], RR.fwd_bits(pkg, v).reshape(-1))
    yf = pkg.bf16_bits_to_f32(y[:n]).reshape(N, O)
    assert np.all(yf[:, 0] == np.inf)
    if O > 2:
        assert np.all(y[:n].reshape(N, O)[:, 1] == 0) and np.isnan(yf[:, -1]).all()
        neg = float((v[:, 2:-1] < 0).mean())
        assert 0.2 < neg < 0.8, neg
    assert not np.any(y[:n] == 0x8000)
    assert np.all(y[n:] == NAN_BF16)
    assert np.array_equal(run_fwd(plan, xd, n), y)
    plan.close()
    print(f"{name}: forward splits {info['fwd_splits']}")


def test_linear_cases_cover_split_and_unsplit(pkg):
    splits = [pkg.linear_info(*c[1:6], *linear_layout(c))["fwd_splits"] for c in LINEAR]
    assert min(splits) == 1 and max(splits) > 1, splits


# ------------------------------------------------------------------------------------------------ 2. forward, act 3 against act 0
def check_against_act0(y3, y0):
    """act 3 = act 0 where act 0 is > 0 or NaN, +0 where act 0 is < 0 (and at +-0); never -0"""
    f0 = torch.from_numpy(y0.view(np.int16)).view(torch.bfloat16).float().numpy()
    keep = (f0 > 0) | np.isnan(f0)
    assert np.array_equal(y3[keep], y0[keep])
    assert np.all(y3[~keep] == 0)
    assert not np.any(y3 == 0x8000)
    return float((f0 < 0).mean())


@pytest.mark.parametrize("case", CONV, ids=[cid(c) for c in CONV])
def test_conv_forward_against_act0(eng, pkg, case):
    N, H, W, C, K, R, S, st, pad, P, Q = conv_geometry(case)
    rng = np.random.default_rng(sum(case) + 1)
    x = rng.uniform(-1, 1, (N, H, W, C)).astype(np.float32)
    f = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    b[-1] = np.nan
    xd = conv_x(pkg, x)
    n = N * P * Q * K
    ys = {}
    for act in (pkg.ACT_NONE, pkg.ACT_RELU):
        plan = conv_plan(pkg, eng, case, f, b, act)
        ys[act] = run_fwd(plan, xd, n)
        plan.close()
    neg = check_against_act0(ys[pkg.ACT_RELU][:n], ys[pkg.ACT_NONE][:n])
    assert 0.2 < neg < 0.8, neg


@pytest.mark.parametrize("case", LINEAR, ids=[c[0] for c in LINEAR])
def test_linear_forward_against_act0(eng, pkg, case):
    _, N, P, Q, C, O, _, _ = case
    pitch, rows = linear_layout(case)
    rng = np.random.default_rng(N + O + 1)
    x = rng.normal(0, 1, (N, P, Q, C)).astype(np.float32)
    w = (rng.uniform(-1, 1, (O, P, Q, C)) / np.sqrt(P * Q * C)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, O).astype(np.float32)
    xd = linear_x(pkg, x, pitch, rows)
    ys = {}
    for act in (pkg.ACT_NONE, pkg.ACT_RELU):
        plan = pkg.LinearPlan(eng, N, P, Q, C, O, w, b, act=act, row_pitch=pitch, image_rows=rows)
        ys[act] = run_fwd(plan, xd, N * O)
        plan.close()
    check_against_act0(ys[pkg.ACT_RELU][:N * O], ys[pkg.ACT_NONE][:N * O])


# ------------------------------------------------------------------------------------------------ 3. pcnn_conv_bias_act_bwd at act 3
BA_THREADS, BA_ITERS = 256, 8
KS = [1, 6, 8, 16, 64, 120, 256]
PIXELS = [1, 7, 1001]
GRID = [(K, p) for K in KS for p in PIXELS] + [(64, 128 * 56 * 56)]
SPECIAL_BITS = np.array([0x0000, 0x8000, 0x7F80, 0xFF80, 0x7FC0, 0xFFC0, 0x0001, 0x8001, 0x3F80, 0xBF80], np.uint16)


def n_acc(pixels, K):
    """longest chain of fp32 additions behind one db[k] (as in test_conv_train_gpu.py)"""
    lanes = BA_THREADS // (K // 8 if K % 8 == 0 else K)
    ctas = -(-pixels // (BA_ITERS * lanes))
    return BA_ITERS + lanes + -(-ctas // 8) + 3


def run_bias_act(eng, y, dy, act, with_db=True, in_place=False):
    pixels, K = dy.shape
    yd, dyd = eng.to_device(y), eng.to_device(dy)
    db = eng.to_device(np.full(K, np.nan, np.float32)) if with_db else None
    dpre = dyd if in_place else eng.to_device(np.full(pixels * K + TAIL, NAN_BF16, np.uint16))
    eng.conv_bias_act_bwd(yd, dyd, dpre, db, pixels, K, act)
    eng.sync()
    return dpre.to_host(), (db.to_host() if with_db else None)


def relu_operands(pkg, rng, pixels, K, special=True):
    """y: half ReLU outputs (>= 0), half any sign; dy normal; both with NaN, +-0, +-Inf and subnormals sprinkled in"""
    yf = rng.standard_normal((pixels, K)).astype(np.float32)
    yf = np.where(rng.random((pixels, K)) < 0.5, np.maximum(yf, 0), yf)
    y, dy = pkg.f32_to_bf16_bits(yf), pkg.f32_to_bf16_bits(rng.standard_normal((pixels, K)).astype(np.float32))
    if special:
        for a in (y, dy):
            flat = a.reshape(-1)
            m = min(flat.size, 3 * SPECIAL_BITS.size)
            idx = rng.choice(flat.size, m, replace=False)
            flat[idx] = np.resize(SPECIAL_BITS, m)
    return y, dy


@pytest.mark.parametrize("K,pixels", GRID, ids=[f"K{K}-px{p}" for K, p in GRID])
def test_bias_act_relu(eng, pkg, K, pixels):
    """dpre bit-identical to the replay on y and dy holding NaN, +-0, +-Inf; db within the fp32 bound of the float64 sum (equal
    where that sum is not finite); NaN-prefilled dpre fully written, its tail untouched; in place = out of place; reruns
    bit-identical; db = NULL gives the same dpre"""
    rng = np.random.default_rng(K * 131 + pixels)
    y, dy = relu_operands(pkg, rng, pixels, K)
    n = pixels * K
    dpre, db = run_bias_act(eng, y, dy, pkg.ACT_RELU)
    want = RR.bwd_bits(pkg, y, dy)
    assert np.array_equal(dpre[:n].reshape(pixels, K), want)
    assert np.all(dpre[n:] == NAN_BF16)
    d64 = pkg.bf16_bits_to_f32(want).astype(np.float64)
    with np.errstate(invalid="ignore"):
        ref = d64.sum(axis=0)
        bound = 2 * n_acc(pixels, K) * 2.0 ** -24 * np.abs(d64).sum(axis=0)
    fin = np.isfinite(ref)
    assert np.all(np.abs(db[fin] - ref[fin]) <= bound[fin])
    assert np.array_equal(np.isnan(db), np.isnan(ref))                  # +-Inf and NaN terms: any order gives the same
    inf = ~fin & ~np.isnan(ref)
    assert np.array_equal(db[inf], ref[inf].astype(np.float32))
    ip, db_ip = run_bias_act(eng, y, dy, pkg.ACT_RELU, in_place=True)
    assert np.array_equal(ip.reshape(pixels, K), want) and np.array_equal(db_ip.view(np.uint32), db.view(np.uint32))
    again, db2 = run_bias_act(eng, y, dy, pkg.ACT_RELU)
    assert np.array_equal(again, dpre) and np.array_equal(db2.view(np.uint32), db.view(np.uint32))
    nodb, _ = run_bias_act(eng, y, dy, pkg.ACT_RELU, with_db=False)
    assert np.array_equal(nodb, dpre)


@pytest.mark.parametrize("K,pixels", GRID, ids=[f"K{K}-px{p}" for K, p in GRID])
def test_bias_act_relu_integer_exact(eng, pkg, K, pixels):
    """y in {-1, -0, 0, 1/2, 1}, dy in -2..2: every partial sum of db is an exact integer, so db is bit-identical to float64"""
    rng = np.random.default_rng(K + 3 * pixels)
    y = rng.choice(np.array([0xBF80, 0x8000, 0x0000, 0x3F00, 0x3F80], np.uint16), (pixels, K))
    dy = pkg.f32_to_bf16_bits(rng.integers(-2, 3, (pixels, K)).astype(np.float32))
    dpre, db = run_bias_act(eng, y, dy, pkg.ACT_RELU)
    want = RR.bwd_bits(pkg, y, dy)
    assert np.array_equal(dpre[:pixels * K].reshape(pixels, K), want)
    assert np.array_equal(db.astype(np.float64), pkg.bf16_bits_to_f32(want).astype(np.float64).sum(axis=0))


def test_relu_refusals(eng, pkg):
    K, pixels = 16, 64
    y, dy, dpre = (eng.array((pixels + 8, K), np.uint16) for _ in range(3))
    db = eng.array(K + 8)
    call = eng.conv_bias_act_bwd
    msg = "pcnn_conv_bias_act_bwd: act {} is not 0 \\(none\\), 1 \\(sigmoid\\) or 3 \\(ReLU\\)"
    for act in (2, 4, -1):
        with pytest.raises(pkg.PcnnError, match=msg.format(act)):
            call(y, dy, dpre, db, pixels, K, act)
    with pytest.raises(pkg.PcnnError, match="act 3 \\(ReLU\\) needs y"):
        call(None, dy, dpre, db, pixels, K, 3)
    with pytest.raises(pkg.PcnnError, match="act 3 \\(ReLU\\) needs y"):
        call(y, dy, None, db, pixels, K, 3)
    with pytest.raises(pkg.PcnnError, match="overlapping"):
        call(y, dy, y, db, pixels, K, 3)
    call(y, dy, dy, None, pixels, K, 3)                                  # in place without a bias is allowed
    eng.sync()
    f = np.zeros((6, 5, 5, 1), np.float32)
    for act in (2, 4, -1):                                              # the row-Toeplitz create call validates act too
        with pytest.raises(pkg.PcnnError, match=f"pcnn_conv_tc_plan_create: act {act} is not 0 \\(none\\), 1 \\(sigmoid\\) or 3"):
            pkg.ConvPlan(eng, 2, 28, 28, 1, 6, 5, 5, f, act=act)
    with pytest.raises(pkg.PcnnError, match="pcnn_conv_wide_plan_create_padded: act 2 is not 0 \\(none\\), 1 \\(sigmoid\\) or 3"):
        pkg.WideConvPlan(eng, 2, 6, 6, 8, 16, 3, 3, np.zeros((16, 3, 3, 8), np.float32), act=2, padding=(1, 1))
    with pytest.raises(pkg.PcnnError, match="pcnn_linear_plan_create: act 4 is not 0 \\(none\\), 1 \\(sigmoid\\) or 3"):
        pkg.LinearPlan(eng, 64, 2, 2, 8, 10, np.zeros((10, 2, 2, 8), np.float32), act=4)
    for a in (y, dy, dpre, db):
        a.free()


# ------------------------------------------------------------------------------------------------ 4. one layer step vs float64
LAYERS = [  # N, H, W, C, K, R, S, stride, pad: one row-Toeplitz and one wide layer
    (8, 28, 28, 1, 8, 5, 5, 1, 0),
    (4, 24, 24, 8, 16, 3, 3, 1, 1),
]


@pytest.mark.parametrize("case", LAYERS, ids=["narrow", "wide"])
def test_conv_layer_step_relu(eng, pkg, case):
    """ConvLayer at act 3 with bias, random operands: y within the fp32 accumulation bound of relu(float64) (ReLU is
    1-Lipschitz), dpre (dy rewritten in place) the replay on the layer's own y, dw, db and dx against float64 on that dpre"""
    N, H, W, C, K, R, S, st, pad = case
    P, Q = (H + 2 * pad - R) // st + 1, (W + 2 * pad - S) // st + 1
    rng = np.random.default_rng(9)
    f32 = pkg.bf16_bits_to_f32
    x = f32(pkg.f32_to_bf16_bits(rng.uniform(0, 1, (N, H, W, C)).astype(np.float32)))
    f = f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    dy = pkg.f32_to_bf16_bits(rng.standard_normal((N, P, Q, K)).astype(np.float32))
    layer = pkg.ConvLayer(eng, N, H, W, C, K, R, S, f, b, act=pkg.ACT_RELU, stride=st, padding=(pad, pad))
    assert layer.family == ("narrow" if pad == 0 else "wide")
    pitch = layer.row_pitch
    xl = np.zeros((N * H, pitch), np.uint16)
    xl[:, :W * C] = pkg.f32_to_bf16_bits(x).reshape(N * H, W * C)
    xd, yd, dyd = eng.to_device(xl), eng.to_device(np.full((N, P, Q, K), NAN_BF16, np.uint16)), eng.to_device(dy)
    dx = eng.to_device(np.full((N * H, pitch), NAN_BF16, np.uint16))
    layer.forward(xd, yd)
    layer.backward(yd, dyd, dx)
    eng.sync()
    y, dpre_bits = yd.to_host(), dyd.to_host()
    xp = np.pad(x.astype(np.float64), ((0, 0), (pad, pad), (pad, pad), (0, 0)))
    pre = CR.conv_fwd_f64(xp, f, b, st)
    pre_abs = CR.conv_fwd_f64(np.abs(xp), np.abs(f), np.abs(b), st)
    ref = RR.relu(pre)
    assert np.all(np.abs(f32(y) - ref) <= 2 * R * S * C * 2.0 ** -24 * pre_abs + 2.0 ** -8 * ref)
    assert 0.1 < float((pre < 0).mean()) < 0.9
    assert np.array_equal(dpre_bits, RR.bwd_bits(pkg, y, dy))
    dpre = f32(dpre_bits).astype(np.float64)
    dw = CS.conv_wgrad_f64(xp, dpre, R, S, st)
    dx_ref = CS.conv_dgrad_f64(dpre, f.astype(np.float64), H + 2 * pad, W + 2 * pad, st)[:, pad:pad + H, pad:pad + W, :]
    dw_abs = CS.conv_wgrad_f64(np.abs(xp), np.abs(dpre), R, S, st)
    dx_abs = CS.conv_dgrad_f64(np.abs(dpre), np.abs(f.astype(np.float64)), H + 2 * pad, W + 2 * pad, st)[:, pad:pad + H, pad:pad + W, :]
    npix = N * P * Q
    assert np.all(np.abs(layer.dw.to_host() - dw) <= 2 * npix * 2.0 ** -24 * dw_abs + 1e-30)
    assert np.all(np.abs(layer.db.to_host() - dpre.sum(axis=(0, 1, 2))) <= 2 * npix * 2.0 ** -24 * np.abs(dpre).sum(axis=(0, 1, 2)))
    got_dx = f32(dx.to_host()[:, :W * C].reshape(N, H, W, C)).astype(np.float64)
    assert np.all(np.abs(got_dx - dx_ref) <= 2.0 ** -8 * np.abs(dx_ref) + 2 * K * R * S * 2.0 ** -24 * dx_abs + 1e-30)
    layer.close()


def test_linear_layer_step_relu(eng, pkg):
    """LinearLayer at act 3 with bias (LeNet fc1's shape), random operands, bounds of test_linear_gpu.py"""
    N, P, Q, C, O, pitch, rows = 128, 6, 6, 16, 128, 96, 6
    rng = np.random.default_rng(13)
    f32 = pkg.bf16_bits_to_f32
    x = f32(pkg.f32_to_bf16_bits(rng.normal(0, 1, (N, P, Q, C)).astype(np.float32)))
    w = rng.uniform(-1, 1, (O, P, Q, C)).astype(np.float32) / np.float32(np.sqrt(P * Q * C))
    b = rng.uniform(-0.5, 0.5, O).astype(np.float32)
    dy_bits = pkg.f32_to_bf16_bits(rng.normal(0, 1, (N, O)).astype(np.float32))
    layer = pkg.LinearLayer(eng, N, P, Q, C, O, w, b, act=pkg.ACT_RELU, row_pitch=pitch, image_rows=rows)
    xd = linear_x(pkg, x, pitch, rows)
    y, dyd, dx = nan_buf(N * O), dev_bits(dy_bits), nan_buf(N * rows * pitch)
    layer.forward(xd, y)
    layer.backward(y, dyd, dx)
    eng.sync()
    yh = host(y).reshape(N, O)
    wb = f32(pkg.f32_to_bf16_bits(w)).astype(np.float64)
    F_ = P * Q * C
    pre = LR.fwd_f64(x, wb, b)
    ref = RR.relu(pre)
    bound = 2 * F_ * 2.0 ** -24 * LR.fwd_f64(np.abs(x), np.abs(wb)) + 1e-30
    assert np.all(np.abs(f32(yh) - ref) <= bound + 2.0 ** -8 * ref)
    assert np.array_equal(host(dyd).reshape(N, O), RR.bwd_bits(pkg, yh, dy_bits))
    d = f32(host(dyd)).astype(np.float64).reshape(N, O)
    assert np.all(np.abs(layer.dw.to_host() - LR.wgrad_f64(x, d)) <= 2 * N * 2.0 ** -24 * LR.wgrad_f64(np.abs(x), np.abs(d)) + 1e-30)
    assert np.all(np.abs(layer.db.to_host() - d.sum(0)) <= 2 * N * 2.0 ** -24 * np.abs(d).sum(0))
    dxh = host(dx).reshape(N, rows, pitch)
    ref_dx = LR.dgrad_f64(d, wb).reshape(N, P, Q * C)
    dxb = 2 * O * 2.0 ** -24 * LR.dgrad_f64(np.abs(d), np.abs(wb)).reshape(N, P, Q * C)
    assert np.all(np.abs(f32(dxh[:, :P, :Q * C]) - ref_dx) <= dxb + 2.0 ** -8 * np.abs(ref_dx) + 1e-30)
    layer.close()


# ------------------------------------------------------------------------------------------------ 5. end to end
ACC_MIN = 0.75          # a float32 torch CPU replica of this network, seed and step reaches 0.844


def test_relu_classifier_mnist(eng, pkg, golden):
    """ReLU in c1, c2 and fc1.  In each of the first 5 steps every ReLU layer's dpre is bit-exact against the replay on the
    device's own y and dy.  A second fresh run reproduces the parameters after 5 steps bit for bit.  After EPOCHS epochs over
    the 1024 training digits the mean loss has fallen and test accuracy on the 256 test digits exceeds ACC_MIN."""

    def check_step(net, it, x, labels):
        net.forward(x, labels)
        seen = {}

        def hook(name, y, dy):
            eng.sync()
            seen[name] = (host(y).copy(), host(dy).copy())
        net.backward(hook)
        eng.sync()
        for name in ("fc1", "c2", "c1"):
            y, dy = seen[name + ":before"]
            dpre = seen[name + ":after"][1]
            assert np.array_equal(dpre, RR.bwd_bits(pkg, y, dy)), (it, name)
            frac = float((pkg.bf16_bits_to_f32(y) > 0).mean())
            assert 0.05 < frac < 0.95, (it, name, frac)          # the layer is neither dead nor linear

    ep_loss, acc, _ = train(eng, pkg, golden, lambda: ReluNet(eng, pkg, ReluNet.init_params()), ReluNet.EPOCHS, check_step=check_step)
    print(f"ReLU classifier: mean loss by epoch {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}; test accuracy {acc:.4f} (threshold {ACC_MIN})")
    assert np.isfinite(ep_loss).all() and ep_loss[-1] < ep_loss[0]
    assert acc > ACC_MIN
