"""Fully connected layers on the device (pcnn_linear_plan_create run by pcnn_conv_tc_fwd, pcnn_linear_wgrad / _dgrad,
LinearPlan, LinearLayer) and the bf16 softmax cross-entropy (pcnn_softmax_ce_bf16), against the float64 references of
linear_ref.py (pinned to torch by test_linear_cpu.py): exact integer operands bit for bit, random operands with bias and sigmoid
within the fp32 accumulation bound, refreshed plans, every refusal, and a LeNet-style classifier trained on MNIST digits."""
import numpy as np
import pytest
import torch

import linear_ref as LR
import maxpool_ref as MR
from example_nets import DEV, NAN_BF16, Net, host, nan_buf, train

pytestmark = pytest.mark.gpu

CASES = [  # id, N, P, Q, C, O, row_pitch (0 = Q*C rounded up to 8), image_rows (0 = P)
    ("n100-qc130-pitched-fwdsplit", 100, 6, 5, 26, 10, 144, 8),
    ("n200-o1", 200, 2, 3, 8, 1, 0, 0),
    ("n33-qc7-pitched", 33, 1, 1, 7, 16, 24, 3),
    ("fc-after-fc-o16", 300, 1, 1, 128, 16, 0, 0),
    ("n257-o120", 257, 3, 3, 24, 120, 0, 0),
    ("n129-o256-qc80", 129, 2, 2, 40, 256, 0, 0),
    ("lenet-fc1", 128, 6, 6, 16, 128, 96, 6),
    ("lenet-fc2", 128, 1, 1, 128, 10, 128, 1),
    ("head-7x7x256-n1024", 1024, 7, 7, 256, 256, 0, 0),
    ("head-1x1x2048-n4096", 4096, 1, 1, 2048, 256, 0, 0),
]


def layout(case):
    _, N, P, Q, C, O, pitch, rows = case
    return (pitch or (Q * C + 7) // 8 * 8), (rows or P)


def dev_bits(bits):
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).to(DEV)


def put_x(pkg, x, pitch, rows):
    """x [N][P][Q][C] (bf16-exact float32) into [N][rows][pitch] with NaN in every pad element"""
    N, P, Q, C = x.shape
    buf = np.full((N, rows, pitch), NAN_BF16, np.uint16)
    buf[:, :P, :Q * C] = pkg.f32_to_bf16_bits(x).reshape(N, P, Q * C)
    return dev_bits(buf)


def run_all(eng, plan, xd, dyd, case):
    _, N, P, Q, C, O, _, _ = case
    pitch, rows = layout(case)
    y, dx = nan_buf(N, O), nan_buf(N, rows, pitch)
    dw = eng.array((O, P, Q, C))
    plan.fwd(xd, y)
    eng.linear_wgrad(plan, xd, dyd, dw)
    eng.linear_dgrad(plan, dyd, dx)
    eng.sync()
    out = host(y), dw.to_host(), host(dx)
    dw.free()
    return out


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_exact_integers(eng, pkg, case):
    """small integer x, W, b and dy: every fp32 partial sum is exact in any order, so y, dW and dx are bit-identical to the
    rounded integer reference; NaN-prefilled outputs are fully written, dx's pad stays NaN, reruns are bit-identical and
    <dy, x W^T> = <dW, W> = <dx, x> exactly where dx is exact in bf16"""
    _, N, P, Q, C, O, _, _ = case
    pitch, rows = layout(case)
    info = pkg.linear_info(N, P, Q, C, O, pitch, rows)
    rng = np.random.default_rng(N + 7 * O)
    x = rng.integers(-3, 4, (N, P, Q, C)).astype(np.float32)
    w = rng.integers(-3, 4, (O, P, Q, C)).astype(np.float32)
    b = rng.integers(-8, 9, O).astype(np.float32)
    dy = rng.integers(-3, 4, (N, O)).astype(np.float32)
    plan = pkg.LinearPlan(eng, N, P, Q, C, O, w, b, act=0, row_pitch=pitch, image_rows=rows)
    xd, dyd = put_x(pkg, x, pitch, rows), dev_bits(pkg.f32_to_bf16_bits(dy))
    y, dw, dx = run_all(eng, plan, xd, dyd, case)
    assert np.array_equal(y, pkg.f32_to_bf16_bits(LR.fwd_f64(x, w, b).astype(np.float32)))
    ref_dw = LR.wgrad_f64(x, dy)
    assert np.array_equal(dw, ref_dw.astype(np.float32))
    ref_dx = LR.dgrad_f64(dy, w)
    assert np.array_equal(dx[:, :P, :Q * C], pkg.f32_to_bf16_bits(ref_dx.astype(np.float32)).reshape(N, P, Q * C))
    assert (dx[:, P:, :] == NAN_BF16).all() and (dx[:, :P, Q * C:] == NAN_BF16).all()
    again = run_all(eng, plan, xd, dyd, case)
    assert all(np.array_equal(a, b_) for a, b_ in zip((y, dw, dx), again))
    inner = float((dy.astype(np.float64) * LR.fwd_f64(x, w)).sum())
    assert float((dw.astype(np.float64) * w).sum()) == inner
    if np.abs(ref_dx).max() <= 256:
        dxf = pkg.bf16_bits_to_f32(dx[:, :P, :Q * C]).astype(np.float64).reshape(N, P, Q, C)
        assert float((dxf * x).sum()) == inner
    plan.close()
    print(case[0], "fwd splits", info["fwd_splits"], "wgrad splits", info["wgrad_splits"])


RANDOM = [  # id, N, P, Q, C, O, row_pitch, image_rows, act, bias
    ("lenet-fc1-sigmoid", 128, 6, 6, 16, 128, 96, 6, 1, True),
    ("n100-qc130-sigmoid", 100, 6, 5, 26, 10, 144, 8, 1, True),
    ("fc2-o10", 128, 1, 1, 128, 10, 128, 1, 0, True),
    ("n300-o24-nobias", 300, 3, 3, 40, 24, 0, 0, 0, False),
    ("head-7x7x256-sigmoid", 1024, 7, 7, 256, 256, 0, 0, 1, True),
]


@pytest.mark.parametrize("case", RANDOM, ids=[c[0] for c in RANDOM])
def test_layer_random(eng, pkg, case):
    """LinearLayer forward and backward on random operands against float64 on the device's bf16 operands: the fp32 accumulation
    bound 2 n 2^-24 sum |terms|, plus one bf16 rounding of y and dx (and the sigmoid's tanh.approx for y)"""
    _, N, P, Q, C, O, pitch, rows, act, with_bias = case
    rng = np.random.default_rng(O * 3 + N)
    f32 = pkg.bf16_bits_to_f32
    x = f32(pkg.f32_to_bf16_bits(rng.normal(0, 1, (N, P, Q, C)).astype(np.float32)))
    w = rng.uniform(-1, 1, (O, P, Q, C)).astype(np.float32) / np.float32(np.sqrt(P * Q * C))
    b = rng.uniform(-0.5, 0.5, O).astype(np.float32) if with_bias else None
    dy = f32(pkg.f32_to_bf16_bits(rng.normal(0, 1, (N, O)).astype(np.float32)))
    layer = pkg.LinearLayer(eng, N, P, Q, C, O, w, b, act=act, row_pitch=pitch, image_rows=rows)
    pitch, rows = layer.row_pitch, layer.image_rows or P
    xd = put_x(pkg, x, pitch, rows)
    y, dyd, dx = nan_buf(N, O), dev_bits(pkg.f32_to_bf16_bits(dy)), nan_buf(N, rows, pitch)
    layer.forward(xd, y)
    eng.sync()
    yh = host(y)
    layer.backward(y, dyd, dx)
    eng.sync()
    wb = f32(pkg.f32_to_bf16_bits(w)).astype(np.float64)
    F_ = P * Q * C
    pre = LR.fwd_f64(x, wb, b)
    bound = 2 * F_ * 2.0 ** -24 * LR.fwd_f64(np.abs(x), np.abs(wb)) + 1e-30
    yf = f32(yh).astype(np.float64)
    if act:
        ref = 1 / (1 + np.exp(-pre))
        assert np.all(np.abs(yf - ref) <= bound / 4 + 2.0 ** -8 * np.abs(ref) + 1e-3)
    else:
        assert np.all(np.abs(yf - pre) <= bound + 2.0 ** -8 * np.abs(pre))
    d = f32(host(dyd)).astype(np.float64)                            # dpre after backward (dy itself without sigmoid)
    if act:
        y32 = f32(yh)
        assert np.array_equal(host(dyd), pkg.f32_to_bf16_bits(dy * (y32 * (np.float32(1) - y32))))
    dw = layer.dw.to_host()
    ref_dw = LR.wgrad_f64(x, d)
    assert np.all(np.abs(dw - ref_dw) <= 2 * N * 2.0 ** -24 * LR.wgrad_f64(np.abs(x), np.abs(d)) + 1e-30)
    if with_bias:
        db = layer.db.to_host()
        assert np.all(np.abs(db - d.sum(0)) <= 2 * N * 2.0 ** -24 * np.abs(d).sum(0))
    dxh = host(dx)
    ref_dx = LR.dgrad_f64(d, wb).reshape(N, P, Q * C)
    dxb = 2 * O * 2.0 ** -24 * LR.dgrad_f64(np.abs(d), np.abs(wb)).reshape(N, P, Q * C)
    assert np.all(np.abs(f32(dxh[:, :P, :Q * C]) - ref_dx) <= dxb + 2.0 ** -8 * np.abs(ref_dx) + 1e-30)
    assert (dxh[:, P:, :] == NAN_BF16).all() and (dxh[:, :P, Q * C:] == NAN_BF16).all()
    layer.close()


def test_refresh_matches_fresh_plan_and_is_stream_ordered(eng, pkg):
    """set_params on a linear plan gives the bits of a plan created from the same parameters, special values included, in
    the forward and the input gradient; a forward enqueued before the refresh reads the old parameters"""
    N, P, Q, C, O = 200, 3, 3, 24, 40
    rng = np.random.default_rng(3)
    w1 = rng.normal(0, 0.1, (O, P, Q, C)).astype(np.float32)
    w2 = rng.normal(0, 0.1, (O, P, Q, C)).astype(np.float32)
    w2.reshape(-1)[:6] = [np.nan, np.inf, -np.inf, -0.0, 3.0e38, 1e-40]
    b1, b2 = rng.normal(size=O).astype(np.float32), rng.normal(size=O).astype(np.float32)
    x = rng.normal(0, 1, (N, P, Q, C)).astype(np.float32)
    xd = put_x(pkg, x, Q * C, P)
    dyd = dev_bits(pkg.f32_to_bf16_bits(rng.normal(size=(N, O)).astype(np.float32)))
    fresh1 = pkg.LinearPlan(eng, N, P, Q, C, O, w1, b1, act=1)
    fresh2 = pkg.LinearPlan(eng, N, P, Q, C, O, w2, b2, act=1)
    plan = pkg.LinearPlan(eng, N, P, Q, C, O, w1, b1, act=1)
    w2d, b2d = eng.to_device(w2), eng.to_device(b2)
    outs = [nan_buf(N, O) for _ in range(4)]
    dxs = [nan_buf(N, P, Q * C) for _ in range(2)]
    fresh1.fwd(xd, outs[0])
    fresh2.fwd(xd, outs[1])
    eng.linear_dgrad(fresh2, dyd, dxs[0])
    plan.fwd(xd, outs[2])                                            # enqueued before the refresh: old parameters
    plan.set_params(w2d, b2d)
    plan.fwd(xd, outs[3])
    eng.linear_dgrad(plan, dyd, dxs[1])
    eng.sync()
    assert np.array_equal(host(outs[2]), host(outs[0]))
    assert np.array_equal(host(outs[3]), host(outs[1]))
    assert np.array_equal(host(dxs[1]), host(dxs[0]))
    assert not np.array_equal(host(outs[3]), host(outs[2]))
    for p_ in (fresh1, fresh2, plan):
        p_.close()


def test_refusals(eng, pkg):
    N, P, Q, C, O = 64, 2, 2, 8, 10
    w = np.zeros((O, P, Q, C), np.float32)
    with pytest.raises(pkg.PcnnError, match="act 2 is not 0"):
        pkg.LinearPlan(eng, N, P, Q, C, O, w, act=2)
    with pytest.raises(pkg.PcnnError, match="1 <= O <= 256"):
        pkg.LinearPlan(eng, N, P, Q, C, 257, np.zeros((257, P, Q, C), np.float32))
    with pytest.raises(pkg.PcnnError, match="hidden width"):
        pkg.LinearPlan(eng, N, 1, 1, 10, O, np.zeros((O, 10), np.float32), row_pitch=10)
    plan = pkg.LinearPlan(eng, N, P, Q, C, O, w)                    # no bias
    x, dy, dx = nan_buf(N, P, Q * C), nan_buf(N, O), nan_buf(N, P, Q * C)
    dw = eng.array((O, P, Q, C))
    with pytest.raises(pkg.PcnnError, match="only a plan with a bias"):
        plan.set_params(None, eng.array(O))
    with pytest.raises(pkg.PcnnError, match="16-byte aligned"):
        eng.linear_wgrad(plan, x.data_ptr() + 2, dy, dw)
    with pytest.raises(pkg.PcnnError, match="16-byte aligned"):
        eng.linear_dgrad(plan, dy, dx.data_ptr() + 2)
    with pytest.raises(pkg.PcnnError, match="16-byte aligned"):
        plan.fwd(x, dy.data_ptr() + 2)
    conv = pkg.WideConvPlan(eng, 2, 6, 6, 8, 16, 3, 3, np.zeros((16, 3, 3, 8), np.float32), padding=(1, 1))
    with pytest.raises(pkg.PcnnError, match="pcnn_linear_wgrad: the plan was not made by pcnn_linear_plan_create"):
        eng.linear_wgrad(conv, x, dy, dw)
    with pytest.raises(pkg.PcnnError, match="pcnn_linear_dgrad: the plan was not made by pcnn_linear_plan_create"):
        eng.linear_dgrad(conv, dy, dx)
    lab = torch.zeros(N, dtype=torch.uint8, device=DEV)
    with pytest.raises(pkg.PcnnError, match="1 <= O <= 256"):
        eng.softmax_ce_bf16(dy, lab, N, 257, 1.0, nan_buf(N, 257))
    with pytest.raises(pkg.PcnnError, match="overlaps logits"):
        eng.softmax_ce_bf16(dy, lab, N, O, 1.0, dy.data_ptr() + 16)
    eng.sync()
    conv.close()
    plan.close()
    dw.free()


@pytest.mark.parametrize("O", [1, 10, 37, 256])
def test_softmax_ce_bf16(eng, pkg, O):
    """dlogits bit-identical to the float64 -> fp32 -> bf16 replay (one bf16 ulp allowed within 1e-12 of a rounding boundary,
    counted), the loss within 1e-6, pred exact with ties, NaN rows and labels >= O; in place gives the same bits"""
    N = 515
    rng = np.random.default_rng(O)
    z = np.where(rng.random((N, O)) < 0.5, rng.integers(-4, 5, (N, O)) / 2.0, rng.normal(0, 3, (N, O))).astype(np.float32)
    z[::7] = rng.integers(-2, 3, (len(z[::7]), O)) / 2.0             # many ties
    z[5, O // 2] = np.nan
    z[11] = -np.inf
    zb = pkg.f32_to_bf16_bits(z)
    labels = rng.integers(0, O, N).astype(np.uint8)
    labels[[3, 17]] = [O, 255] if O < 255 else [255, 255]
    scale = 1.0 / N
    zd, lab = dev_bits(zb), torch.from_numpy(labels).to(DEV)
    d = nan_buf(N, O)
    loss = torch.full((N,), float("nan"), dtype=torch.float32, device=DEV)
    pred = torch.full((N,), -7, dtype=torch.int32, device=DEV)
    eng.softmax_ce_bf16(zd, lab, N, O, scale, d, loss, pred)
    eng.sync()
    g, lref, pref = LR.softmax_ce_f64(pkg.bf16_bits_to_f32(zb), labels, np.float32(scale))
    dh = host(d)
    nan = np.isnan(g)
    assert np.array_equal(np.isnan(pkg.bf16_bits_to_f32(dh)), nan)
    exp = LR.f64_to_bf16_bits(pkg, np.where(nan, 0, g))
    diff = np.abs(dh.astype(np.int64) - exp.astype(np.int64))
    near = LR.near_boundary(pkg, np.where(nan, 0, g)) & ~nan
    assert np.all((diff[~nan] == 0) | (near[~nan] & (diff[~nan] <= 1)))
    print(f"O = {O}: {int(near.sum())} values near a rounding boundary, {int((diff[~nan] != 0).sum())} one ulp off")
    lh = loss.cpu().numpy()
    assert np.array_equal(np.isnan(lh), np.isnan(lref))
    ok = ~np.isnan(lref)
    assert np.all(np.abs(lh[ok] - lref[ok]) <= 1e-6 * np.maximum(1.0, np.abs(lref[ok])))
    assert np.array_equal(pred.cpu().numpy(), pref)
    assert pref[5] == -1 and pref[11] == 0
    # in place, without loss and pred
    eng.softmax_ce_bf16(zd, lab, N, O, scale, zd)
    eng.sync()
    assert np.array_equal(host(zd), dh)


# ============================================================ end to end: a LeNet-style classifier on MNIST digits
ACC_MIN = 0.70          # the float32 torch replica of this network, seed and step reaches 0.836 (see DESIGN 3.13)


def test_classifier_mnist(eng, pkg, golden):
    """The whole network on the context's stream.  In each of the first 5 steps: both pools bit-exact against the numpy
    reference, dW, db and dx of both linear layers against float64 on the device's own intermediates within the fp32 bound.
    A second fresh run reproduces the parameters after 5 steps bit for bit.  After EPOCHS epochs over the 1024 training digits
    the mean loss has fallen and test accuracy on the 256 test digits exceeds ACC_MIN."""
    f32 = pkg.bf16_bits_to_f32
    B = Net.NB

    def bound_ok(got, ref, absref, n):
        return np.all(np.abs(got - ref) <= 2 * n * 2.0 ** -24 * absref + 1e-30)

    def check_step(net, it, x, labels):
        net.forward(x, labels)
        eng.sync()
        h = {k: host(getattr(net, k)) for k in ("y1", "x2", "y2", "x3", "y3", "z", "dz")}
        h["am1"], h["am2"] = net.p1.argmax.to_host(), net.p2.argmax.to_host()
        w3 = f32(pkg.f32_to_bf16_bits(net.fc1.params()[0])).astype(np.float64)
        w4 = f32(pkg.f32_to_bf16_bits(net.fc2.params()[0])).astype(np.float64)

        def hook(name):
            eng.sync()
            if name == "fc2":
                h["dy3"] = host(net.dy3)
            else:
                h["dpre3"], h["dx3"] = host(net.dy3), host(net.dx3)
        net.backward(hook)
        eng.sync()
        h["dy2"], h["dy1"] = host(net.dy2), host(net.dy1)
        a1 = MR.fwd_argmax(f32(h["y1"]), 2, 2, 2, 0, 0)
        assert np.array_equal(h["am1"], a1) and np.array_equal(h["x2"][:, :, :96].reshape(B, 12, 12, 8), MR.gather(h["y1"], a1, 2, 2, 0, 0))
        a2 = MR.fwd_argmax(f32(h["y2"]), 2, 2, 2, 0, 0)
        assert np.array_equal(h["am2"], a2) and np.array_equal(h["x3"].reshape(B, 6, 6, 16), MR.gather(h["y2"], a2, 2, 2, 0, 0))
        assert np.array_equal(h["dy2"], MR.bwd_bf16(pkg, h["dx3"].reshape(B, 6, 6, 16), a2, 12, 12, 2, 2, 2, 0, 0)), it
        # fc2: x = y3, dy = dz (no sigmoid)
        x4, d4 = f32(h["y3"]).astype(np.float64).reshape(B, 1, 1, 128), f32(h["dz"]).astype(np.float64)
        assert bound_ok(net.fc2.dw.to_host(), LR.wgrad_f64(x4, d4), LR.wgrad_f64(np.abs(x4), np.abs(d4)), B), it
        assert bound_ok(net.fc2.db.to_host(), d4.sum(0), np.abs(d4).sum(0), B), it
        ref = LR.dgrad_f64(d4, w4).reshape(B, 128)
        got = f32(h["dy3"]).astype(np.float64)
        assert np.all(np.abs(got - ref) <= 2 * 10 * 2.0 ** -24 * LR.dgrad_f64(np.abs(d4), np.abs(w4)).reshape(B, 128) + 2.0 ** -8 * np.abs(ref)), it
        # fc1: x = x3 (pool 2's output), dy = dpre3; dx into the pool's dy
        x3, d3 = f32(h["x3"]).astype(np.float64).reshape(B, 6, 6, 16), f32(h["dpre3"]).astype(np.float64)
        assert bound_ok(net.fc1.dw.to_host(), LR.wgrad_f64(x3, d3), LR.wgrad_f64(np.abs(x3), np.abs(d3)), B), it
        assert bound_ok(net.fc1.db.to_host(), d3.sum(0), np.abs(d3).sum(0), B), it
        ref = LR.dgrad_f64(d3, w3).reshape(B, 6, 96)
        got = f32(h["dx3"]).astype(np.float64)
        assert np.all(np.abs(got - ref) <= 2 * 128 * 2.0 ** -24 * LR.dgrad_f64(np.abs(d3), np.abs(w3)).reshape(B, 6, 96) + 2.0 ** -8 * np.abs(ref)), it

    ep_loss, acc, _ = train(eng, pkg, golden, lambda: Net(eng, pkg, Net.init_params()), Net.EPOCHS, check_step=check_step)
    print(f"mean loss by epoch: {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}; test accuracy {acc:.4f} (threshold {ACC_MIN})")
    assert ep_loss[-1] < ep_loss[0]
    assert acc > ACC_MIN
