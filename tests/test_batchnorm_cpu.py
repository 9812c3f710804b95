"""Host-side parts of batch normalization (no GPU): the float64 references of batchnorm_ref.py agree with
torch.nn.functional.batch_norm (training and eval, running statistics included), the residual add and the ReLU, and with torch's
autograd through all three; the float32 replays stay within bf16 rounding of them; pcnn_batchnorm_nhwc_info accepts exactly the
stated domain, reports the partition, and names every rule it refuses."""
import numpy as np
import pytest
import torch

import batchnorm_ref as BR

F = torch.nn.functional


def torch_fwd(x, gamma, beta, r, act, training, eps, momentum, rm, rv):
    """F.batch_norm (+ r) (+ relu) in float64 on [M][C] viewed as [M][C][1][1]"""
    xt = torch.from_numpy(x).reshape(*x.shape, 1, 1)
    rmt, rvt = torch.from_numpy(rm.copy()), torch.from_numpy(rv.copy())
    v = F.batch_norm(xt, rmt, rvt, torch.from_numpy(gamma), torch.from_numpy(beta), training=training, momentum=momentum, eps=eps)
    if r is not None:
        v = v + torch.from_numpy(r).reshape(*r.shape, 1, 1)
    if act == 3:
        v = torch.relu(v)
    return v.reshape(x.shape).numpy(), rmt.numpy(), rvt.numpy()


SHAPES = [(2, 1), (7, 6), (33, 8), (100, 16), (257, 3), (64, 120)]


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("with_r", [False, True])
@pytest.mark.parametrize("act", [0, 3])
@pytest.mark.parametrize("M,C", SHAPES, ids=[f"M{m}-C{c}" for m, c in SHAPES])
def test_forward_reference_matches_torch(M, C, act, with_r, training):
    rng = np.random.default_rng(M * 7 + C + act + 2 * with_r + 5 * training)
    x = rng.standard_normal((M, C)) * rng.uniform(0.5, 3, C) + rng.uniform(-5, 5, C)
    gamma, beta = rng.uniform(0.5, 1.5, C), rng.uniform(-0.5, 0.5, C)
    r = rng.standard_normal((M, C)) if with_r else None
    rm, rv = rng.uniform(-1, 1, C), rng.uniform(0.5, 2, C)
    eps, mom = 1e-5, 0.1
    y, mean, var, rm2, rv2 = BR.fwd_f64(x, gamma, beta, r, act, training, eps, mom, rm, rv)
    yt, rmt, rvt = torch_fwd(x, gamma, beta, r, act, training, eps, mom, rm, rv)
    assert np.allclose(y, yt, rtol=1e-12, atol=1e-12)
    assert np.allclose(rm2, rmt, rtol=1e-12, atol=1e-14) and np.allclose(rv2, rvt, rtol=1e-12, atol=1e-14)
    if training:
        assert np.allclose(mean, x.mean(0)) and np.allclose(var, x.var(0))


@pytest.mark.parametrize("with_dy2", [False, True])
@pytest.mark.parametrize("with_r", [False, True])
@pytest.mark.parametrize("act", [0, 3])
@pytest.mark.parametrize("M,C", SHAPES, ids=[f"M{m}-C{c}" for m, c in SHAPES])
def test_backward_reference_matches_autograd(M, C, act, with_r, with_dy2):
    """bwd_f64 = torch autograd of relu(batch_norm(x) + r) with the incoming gradient dy + dy2: dx, dgamma, dbeta and dr"""
    rng = np.random.default_rng(M * 11 + C + act + 2 * with_r + 4 * with_dy2)
    x = rng.standard_normal((M, C)) * 2 + rng.uniform(-3, 3, C)
    gamma, beta = rng.uniform(0.5, 1.5, C), rng.uniform(-0.5, 0.5, C)
    r = rng.standard_normal((M, C)) if with_r else None
    dy, dy2 = rng.standard_normal((M, C)), (rng.standard_normal((M, C)) if with_dy2 else None)
    y = BR.fwd_f64(x, gamma, beta, r, act)[0]
    dx, dg, db, dr = BR.bwd_f64(x, gamma, y, dy, dy2, act)
    xt = torch.from_numpy(x).reshape(M, C, 1, 1).requires_grad_(True)
    gt, bt = torch.from_numpy(gamma).requires_grad_(True), torch.from_numpy(beta).requires_grad_(True)
    rt = None if r is None else torch.from_numpy(r).reshape(M, C, 1, 1).requires_grad_(True)
    v = F.batch_norm(xt, None, None, gt, bt, training=True, eps=1e-5)
    if rt is not None:
        v = v + rt
    if act == 3:
        v = torch.relu(v)
    assert np.allclose(v.detach().reshape(M, C).numpy(), y, rtol=1e-12, atol=1e-12)
    v.backward(torch.from_numpy(dy + (0 if dy2 is None else dy2)).reshape(M, C, 1, 1))
    assert np.allclose(xt.grad.reshape(M, C).numpy(), dx, rtol=1e-9, atol=1e-11)
    assert np.allclose(gt.grad.numpy(), dg, rtol=1e-10, atol=1e-11) and np.allclose(bt.grad.numpy(), db, rtol=1e-10, atol=1e-11)
    if rt is not None:
        assert np.allclose(rt.grad.reshape(M, C).numpy(), dr, rtol=1e-12, atol=1e-14)


def test_float32_replays_track_float64(pkg):
    """the replays, fed float64 statistics rounded to fp32, stay within a few bf16 ulps of the float64 results"""
    rng = np.random.default_rng(3)
    M, C = 300, 16
    f32 = pkg.bf16_bits_to_f32
    xb = pkg.f32_to_bf16_bits((rng.standard_normal((M, C)) * 2 + 10).astype(np.float32))
    rb = pkg.f32_to_bf16_bits(rng.standard_normal((M, C)).astype(np.float32))
    gamma, beta = rng.uniform(0.5, 1.5, C).astype(np.float32), rng.uniform(-0.5, 0.5, C).astype(np.float32)
    x = f32(xb).astype(np.float64)
    y64, mean, var, _, _ = BR.fwd_f64(x, gamma, beta, f32(rb), 3)
    rstd = (1 / np.sqrt(var + 1e-5)).astype(np.float32)
    yb = BR.fwd_bits(pkg, xb, gamma, beta, mean.astype(np.float32), rstd, rb, 3)
    assert np.all(np.abs(f32(yb) - y64) <= 2.0 ** -7 * (np.abs(y64) + 1) + 1e-30)
    dyb = pkg.f32_to_bf16_bits(rng.standard_normal((M, C)).astype(np.float32))
    g = BR.grad_bits(pkg, yb, dyb, None, 3)
    assert np.array_equal(g, np.where(f32(yb) <= 0, 0, dyb))
    dx64, dg, db, _ = BR.bwd_f64(x, gamma, f32(yb), f32(dyb), None, 3)
    dxb = BR.dx_bits(pkg, xb, g, gamma, mean.astype(np.float32), rstd, dg.astype(np.float32), db.astype(np.float32))
    scale = np.abs(gamma * rstd) * (np.abs(f32(g)) + np.abs(db) / M + np.abs(dg) / M * np.abs((x - mean) * rstd))
    assert np.all(np.abs(f32(dxb) - dx64) <= 2.0 ** -7 * scale + 1e-30)
    assert np.array_equal(BR.running_update(np.ones(C, np.float32), np.zeros(C, np.float32), 0.1), np.full(C, np.float32(0.9)))
    assert BR.eval_rstd(np.float32(4.0), 0.0) == np.float32(0.5)


# ------------------------------------------------------------------------------------------------ pcnn_batchnorm_nhwc_info
def domain_refusal(pixels, C, training):
    if training not in (0, 1):
        return "0 (eval) or 1 (training) is required"
    if not 1 <= C <= 256:
        return "1 <= C <= 256 is required"
    if training and pixels < 2:
        return "training needs more than 1 value per channel"
    if not training and pixels < 1:
        return "at least one pixel"
    return None


def test_info_domain_grid(pkg):
    from ctypes import c_int
    counts = {"accepted": 0, "refused": 0}
    for C in list(range(-1, 20)) + [24, 63, 64, 120, 128, 200, 255, 256, 257, 1000]:
        for pixels in (-1, 0, 1, 2, 3, 7, 1001, 128 * 56 * 56, 1 << 34):
            for training in (0, 1):
                rule = domain_refusal(pixels, C, training)
                try:
                    info = pkg.batchnorm_nhwc_info(pixels, C, training)
                except pkg.PcnnError as e:
                    assert rule is not None and rule in e.msg and "pcnn_batchnorm_nhwc_info" in e.msg, (pixels, C, training, e.msg)
                    counts["refused"] += 1
                    continue
                assert rule is None, (pixels, C, training)
                counts["accepted"] += 1
                vec = 8 if C % 8 == 0 else 1
                lanes = 256 // (C // vec)
                ctas = -(-pixels // (16 * lanes))
                assert info == dict(vec=vec, lanes=lanes, pixels_per_cta=16 * lanes, stat_slots=ctas if training else 0, grad_slots=ctas)
    assert counts["accepted"] > 200 and counts["refused"] > 100, counts
    out = (c_int * 5)()
    assert pkg.lib().pcnn_batchnorm_nhwc_info(10, 8, 2, out) != 0
    assert "training = 2: 0 (eval) or 1 (training) is required" in pkg.lib().pcnn_last_error_string().decode()
    assert pkg.lib().pcnn_batchnorm_nhwc_info(10, 8, 1, None) != 0
    assert "NULL out5" in pkg.lib().pcnn_last_error_string().decode()


def test_info_refusal_messages(pkg):
    info = pkg.batchnorm_nhwc_info
    cases = [
        (lambda: info(10, 0), "pcnn_batchnorm_nhwc_info: C = 0 channels: 1 <= C <= 256 is required"),
        (lambda: info(10, 257), "C = 257 channels: 1 <= C <= 256 is required"),
        (lambda: info(1, 8), "pixels = 1: training needs more than 1 value per channel (pixels = N * H * W >= 2)"),
        (lambda: info(0, 8, False), "pixels = 0: at least one pixel (N * H * W) is required"),
        (lambda: info(1 << 50, 1), "pixels exceed the grid"),
    ]
    for fn, msg in cases:
        with pytest.raises(pkg.PcnnError, match=msg.replace("(", r"\(").replace(")", r"\)").replace("*", r"\*").replace("+", r"\+")):
            fn()
    assert info(1, 8, False) == dict(vec=8, lanes=256, pixels_per_cta=4096, stat_slots=0, grad_slots=1)
    assert info(128 * 56 * 56, 64) == dict(vec=8, lanes=32, pixels_per_cta=512, stat_slots=784, grad_slots=784)
    assert info(1001, 6)["vec"] == 1 and info(1001, 6)["lanes"] == 42
