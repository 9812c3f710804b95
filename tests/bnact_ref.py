"""References of the activations batch normalization fuses besides ReLU (codes 4 SiLU, 5 hard-swish, 6 ReLU6 of
pcnn_batchnorm_nhwc_bf16_fwd and pcnn_batchnorm_nhwc_bf16_bwd_preact):

- float64: act_f64 / dact_f64 and the whole block block_f64 (BN + r + act and its gradients, in the layer's backward order), which
  test_bnact_cpu.py pins to torch's CPU float64 F.silu / F.hardswish / F.relu6 and autograd;
- numpy float32 replays of include/pcnn.h, every operation rounded as the kernels round it: exp_f32 (E), pre32 (the
  pre-activation v), act_bits (y) and grad_bits (g, which is also dr).

numpy float32 arithmetic, "/" included, is IEEE round to nearest with no contraction, which is what the kernels use."""
import numpy as np

import batchnorm_ref as BR

F32 = np.float32
SILU, HARDSWISH, RELU6 = 4, 5, 6
CODES = (SILU, HARDSWISH, RELU6)
NAMES = {SILU: "SiLU", HARDSWISH: "hard-swish", RELU6: "ReLU6"}

# E: the constants of include/pcnn.h, by bit pattern
_f = lambda u: np.array([u], np.uint32).view(F32)[0]
LOG2E, LN2_HI, LN2_LO = _f(0x3FB8AA3B), _f(0x3F317200), _f(0x35BFBE8E)
POLY = [_f(u) for u in (0x3F800000, 0x3F800000, 0x3EFFFFFE, 0x3E2AAA0C, 0x3D2AAC12, 0x3C0933ED, 0x3AB5736C)]   # c0 .. c6
E_HI, E_LO = _f(0x42B17217), _f(0xC2CFF1B4)   # x > E_HI gives +Inf, x < E_LO gives +0
E_MAX_ULP = 1.30                              # the bound pcnn.h states (measured 1.2965 over the finite inputs)


# ------------------------------------------------------------------------------------------------ float32 replays
def exp_f32(x):
    """E(x), the kernels' exponential: k = rint(RN(x log2e)); r = RN(RN(x - RN(k ln2_hi)) - RN(k ln2_lo)); p = the Horner
    polynomial c6 .. c0 in r, each step RN(RN(p r) + c); E = RN(RN(p 2^k1) 2^k2), k1 = floor(k / 2), k2 = k - k1"""
    x = np.asarray(x, F32)
    with np.errstate(all="ignore"):
        k = np.rint(x * LOG2E)
        r = (x - k * LN2_HI) - k * LN2_LO
        p = POLY[-1] * np.ones_like(r)
        for c in POLY[-2::-1]:
            p = p * r + c
        ki = np.clip(np.nan_to_num(k, nan=0.0), -200, 200).astype(np.int64)
        k1 = ki >> 1
        k2 = ki - k1
        out = (p * ((k1 + 127) << 23).astype(np.uint32).view(F32)) * ((k2 + 127) << 23).astype(np.uint32).view(F32)
    out = np.where(x > E_HI, F32(np.inf), out)
    return np.where(x < E_LO, F32(0), out).astype(F32)


def pre32(pkg, x_bits, gamma, beta, mean, rstd, r_bits=None):
    """v = RN(RN(xhat gamma) + beta) (+ float(r)), xhat = RN(RN(float(x) - mean) rstd): the pre-activation of the forward"""
    v = BR.xhat32(pkg, x_bits, mean, rstd) * np.asarray(gamma, F32) + np.asarray(beta, F32)
    return v if r_bits is None else v + pkg.bf16_bits_to_f32(r_bits)


def act32(v, code):
    """act(v) in fp32, before the one bf16 rounding"""
    v = np.asarray(v, F32)
    with np.errstate(all="ignore"):
        if code == SILU:
            return v / (F32(1) + exp_f32(-v))
        if code == HARDSWISH:
            u = v + F32(3)
            u = np.where(u < 0, F32(0), u)
            u = np.where(u > 6, F32(6), u)
            return ((v * u) / F32(6)).astype(F32)
        if code == RELU6:
            u = np.where(v < 0, F32(0), v)
            return np.where(u > 6, F32(6), u).astype(F32)
    raise ValueError(code)


def act_bits(pkg, v, code):
    return pkg.f32_to_bf16_bits(act32(v, code))


def grad_bits(pkg, v, dy_bits, dy2_bits=None, code=SILU):
    """g bits at the pre-activation v: t = float(dy) or RN(float(dy) + float(dy2)); a multiplied derivative d gives
    bf16_rn(RN(t d)), a passed t bf16_rn(t) (dy's bits without dy2), a cut one +0"""
    v = np.asarray(v, F32)
    f32 = pkg.bf16_bits_to_f32
    t = f32(dy_bits) if dy2_bits is None else f32(dy_bits) + f32(dy2_bits)
    passed = np.asarray(dy_bits, np.uint16) if dy2_bits is None else pkg.f32_to_bf16_bits(t)
    zero = np.uint16(0)
    with np.errstate(all="ignore"):
        if code == RELU6:
            return np.where((v > 0) & (v < 6), passed, zero).astype(np.uint16)
        if code == HARDSWISH:
            d = v / F32(3) + F32(0.5)
            g = pkg.f32_to_bf16_bits(t * d)
            return np.where(v <= -3, zero, np.where(v >= 3, passed, g)).astype(np.uint16)
        if code == SILU:
            s = F32(1) / (F32(1) + exp_f32(-v))
            d = s * (F32(1) + v * (F32(1) - s))
            return pkg.f32_to_bf16_bits(t * d)
    raise ValueError(code)


# ------------------------------------------------------------------------------------------------ float64
def act_f64(v, code):
    """torch's CPU formulas: x / (1 + exp(-x)), x * min(max(x + 3, 0), 6) / 6, min(max(x, 0), 6) with NaN passing"""
    v = np.asarray(v, np.float64)
    with np.errstate(all="ignore"):
        if code == SILU:
            return v / (1 + np.exp(-v))
        if code == HARDSWISH:
            u = v + 3
            u = np.where(u < 0, 0.0, u)
            return v * np.where(u > 6, 6.0, u) / 6
        if code == RELU6:
            u = np.where(v < 0, 0.0, v)
            return np.where(u > 6, 6.0, u)
    raise ValueError(code)


def dact_f64(v, t, code):
    """the gradient at v given the incoming t: silu_backward t s (1 + v (1 - s)); hardswish_backward (0 at v <= -3, t at v >= 3,
    t (v / 3 + 1/2) between, NaN at NaN as torch's vectorised loop); hardtanh_backward (t where 0 < v < 6, else 0, NaN included)"""
    v, t = np.asarray(v, np.float64), np.asarray(t, np.float64)
    with np.errstate(all="ignore"):
        if code == SILU:
            s = 1 / (1 + np.exp(-v))
            return t * (s * (1 + v * (1 - s)))
        if code == HARDSWISH:
            return np.where(v <= -3, 0.0, np.where(v >= 3, t, t * (v / 3 + 0.5)))
        if code == RELU6:
            return np.where((v > 0) & (v < 6), t, 0.0)
    raise ValueError(code)


def block_f64(x, gamma, beta, r, dy, dy2, code, eps=1e-5):
    """A training BN + r + act over [M][C] and its backward in the layer's order: y, then g = act'(v) * (dy + dy2) (the
    gradient of r), then dx, dgamma and dbeta from g as batch_norm's backward"""
    y, mean, var, _, _ = BR.fwd_f64(x, gamma, beta, None, 0, eps=eps)
    v = y if r is None else y + np.asarray(r, np.float64)
    t = np.asarray(dy, np.float64) + (0 if dy2 is None else np.asarray(dy2, np.float64))
    g = dact_f64(v, t, code)
    dx, dgamma, dbeta, _ = BR.bwd_f64(x, gamma, None, g, None, 0, eps=eps)
    return act_f64(v, code), v, dx, dgamma, dbeta, g
