"""References of the variational-autoencoder operations (TEST INFRASTRUCTURE ONLY): numpy float32 replays of include/pcnn.h's
log1p_f32 and sincos_2pi_f32, of the Philox Box-Muller normals, of the Gaussian latent (pcnn_gaussian_latent_bf16_fwd / _bwd) and
of the binary cross-entropy with logits (pcnn_bce_logits_bf16), every operation rounded where the kernels round it, so the device
must give their bits.  test_vae_cpu.py pins them to float64 and to torch's float64 autograd.

numpy float32 arithmetic, "/" included, is IEEE round to nearest with no contraction, which is what the kernels use."""
import numpy as np

from bnact_ref import exp_f32
from dropout_ref import LO, S32, philox4x32_10
from restore_ref import bf16_bits, bits_f32

F32 = np.float32
_f = lambda u: np.array([u], np.uint32).view(F32)[0]

# log1p_f32: the constants of include/pcnn.h, by bit pattern
LN2_HI, LN2_LO = _f(0x3F317180), _f(0x3717F7D1)
LG1, LG2, LG3, LG4 = _f(0x3F2AAAAA), _f(0x3ECCCCE1), _f(0x3E91E9EE), _f(0x3E789E26)
SQRT_HALF_BITS = 0x3F3504F3
# sincos_2pi_f32: sin(pi t / 4) = t S(t^2), cos(pi t / 4) = C(t^2) on 0 <= t <= 1
SIN_C = [_f(u) for u in (0x3F490FDB, 0xBDA55DE7, 0x3B2335DE, 0xB81965B4, 0x34A60075)]              # s0 .. s4
COS_C = [_f(u) for u in (0x3F800000, 0xBE9DE9E6, 0x3C81E0F8, 0xB9AAE9DE, 0x3670F449, 0xB2D08CC9)]  # c0 .. c5
LOG1P_MAX_ULP = 0.92         # the bounds pcnn.h states (measured 0.8684 over the Box-Muller inputs, 0.9154 on [0, 1])
SINCOS_MAX_ULP = 1.72        # (measured 1.7154 for each over all 2^24 inputs)
U24 = F32(2.0 ** -24)
GL_DOMAIN = 0xE0000000        # word 1 of every latent counter: the top byte no other draw of the library uses


def ulp_error(got, exact):
    """|got - exact| in fp32 ulps of the float64 exact value (ulp(y) = 2^(floor(log2 |y|) - 23), normal range); at exact == 0
    the error is 0 when got is a zero and +inf otherwise"""
    y, g = np.asarray(exact, np.float64), np.asarray(got, np.float64)
    a = np.abs(y)
    ulp = np.exp2(np.maximum(np.floor(np.log2(np.where(a > 0, a, 1.0))), -126) - 23)
    return np.where(a > 0, np.abs(g - y) / ulp, np.where(g == 0, 0.0, np.inf))


def log1p_f32(e):
    """log1p(e) for float32 e in (-1, 1]: u = RN(1 + e), c = RN(e - RN(u - 1)) (the exact rounding error of u); u = 2^k m with
    m in [sqrt(1/2), sqrt(2)) from u's bits, f = m - 1 (exact); s = f / (2 + f), z = s s, w = z z, R = z (Lg1 + w Lg3) + w (Lg2 +
    w Lg4), hfsq = RN(0.5 f) f; lo = RN(k ln2_lo) + RN(c / u); result ((((s (hfsq + R)) + lo) - hfsq) + f) + RN(k ln2_hi)"""
    e = np.asarray(e, F32)
    with np.errstate(all="ignore"):
        u = F32(1) + e
        c = e - (u - F32(1))
        ix = u.view(np.uint32).astype(np.int64) + (0x3F800000 - SQRT_HALF_BITS)
        k = ((ix >> 23) - 0x7F).astype(F32)
        m = ((ix & 0x7FFFFF) + SQRT_HALF_BITS).astype(np.uint32).view(F32)
        f = m - F32(1)
        s = f / (F32(2) + f)
        z = s * s
        w = z * z
        t1 = w * (LG2 + w * LG4)
        t2 = z * (LG1 + w * LG3)
        R = t2 + t1
        hfsq = (F32(0.5) * f) * f
        lo = k * LN2_LO + c / u
        return (((s * (hfsq + R) + lo) - hfsq) + f + k * LN2_HI).astype(F32)


def sincos_2pi_f32(k):
    """(sin, cos) of 2 pi u, u = k 2^-24, for integer k in [0, 2^24): octant o = k >> 21, j = k & (2^21 - 1); t = j 2^-21 for
    even o and (2^21 - j) 2^-21 for odd o (exact); S = t RN-Horner(s4 .. s0 in t^2), C = RN-Horner(c5 .. c0 in t^2); the octant
    picks (sin, cos) among (+-S, +-C) exactly: o 0 (S, C), 1 (C, S), 2 (C, -S), 3 (S, -C), 4 (-S, -C), 5 (-C, -S), 6 (-C, S),
    7 (-S, C)"""
    k = np.asarray(k, np.int64)
    o, j = k >> 21, k & ((1 << 21) - 1)
    t = (np.where(o & 1, (1 << 21) - j, j).astype(F32) * F32(2.0 ** -21)).astype(F32)
    z = t * t
    p = np.full_like(z, SIN_C[-1])
    for c in SIN_C[-2::-1]:
        p = p * z + c
    S = t * p
    q = np.full_like(z, COS_C[-1])
    for c in COS_C[-2::-1]:
        q = q * z + c
    C = q
    swap = ((o + 1) >> 1) & 1                           # octants 1, 2, 5, 6 take (C, S)
    a, b = np.where(swap, C, S), np.where(swap, S, C)
    sin = np.where(o >= 4, -a, a)
    cos = np.where((o >= 2) & (o <= 5), -b, b)
    return sin.astype(F32), cos.astype(F32)


def box_muller(wa, wb):
    """(n0, n1) of a word pair: u1 = ((wa >> 8) + 1) 2^-24, k2 = wb >> 8; rad = sqrt_rn(RN(-2 log1p_f32(RN(u1 - 1)))),
    n0 = RN(rad cos(2 pi k2 2^-24)), n1 = RN(rad sin(...))"""
    wa, wb = np.asarray(wa, np.uint32), np.asarray(wb, np.uint32)
    u1 = ((wa >> 8).astype(np.int64) + 1).astype(F32) * U24
    rad = np.sqrt(F32(-2) * log1p_f32(u1 - F32(1)))          # numpy's float32 sqrt is correctly rounded, as sqrt_rn
    sn, cs = sincos_2pi_f32((wb >> 8).astype(np.int64))
    return (rad * cs).astype(F32), (rad * sn).astype(F32)


def normals_blocks(q, seed, call):
    """the four normals [..., 4] of Philox block q (uint64 array): counter (q lo, 0xE0000000 | q hi, call lo, call hi), key seed"""
    q = np.asarray(q, np.uint64)
    w = philox4x32_10((q & LO, np.uint64(GL_DOMAIN) | (q >> S32), call & 0xFFFFFFFF, call >> 32), (seed & 0xFFFFFFFF, seed >> 32))
    n0, n1 = box_muller(w[..., 0], w[..., 1])
    n2, n3 = box_muller(w[..., 2], w[..., 3])
    return np.stack([n0, n1, n2, n3], -1)


def eps(R, L, seed, call):
    """epsilon [R][L] float32: element (r, j) is normal (r L + j) & 3 of block (r L + j) >> 2"""
    n = R * L
    q = np.arange(-(-n // 4), dtype=np.uint64)
    return normals_blocks(q, seed, call).reshape(-1)[:n].reshape(R, L)


def _stats(stats_bits, R, L, ld):
    s = bits_f32(np.asarray(stats_bits, np.uint16).reshape(-1)[:R * ld].reshape(R, ld))
    return s[:, :L], s[:, L:2 * L]


def kl_rows(mu, lv):
    """kl [R] float32: RN(0.5 sum), the sum from +0 in ascending j of RN(RN(RN(RN(mu mu) + E(lv)) - 1) - lv)"""
    with np.errstate(all="ignore"):
        term = ((mu * mu + exp_f32(lv)) - F32(1)) - lv
        s = np.zeros(mu.shape[0], F32)
        for j in range(mu.shape[1]):
            s = s + term[:, j]
        return (F32(0.5) * s).astype(F32)


def latent_fwd(stats_bits, R, L, seed, call, ld=None, training=True):
    """(z bits [R][L], kl float32 [R]) of the forward on bf16 stats bits [R][ld] (None = 2L): training z = bf16_rn(RN(mu +
    RN(E(RN(0.5 lv)) eps))), eval z = mu (bits)"""
    ld = 2 * L if ld is None else ld
    mu, lv = _stats(stats_bits, R, L, ld)
    if training:
        with np.errstate(all="ignore"):
            z = bf16_bits(mu + exp_f32(F32(0.5) * lv) * eps(R, L, seed, call))
    else:
        z = np.asarray(stats_bits, np.uint16).reshape(-1)[:R * ld].reshape(R, ld)[:, :L].copy()
    return z, kl_rows(mu, lv)


def latent_bwd(stats_bits, dz_bits, R, L, seed, call, kl_scale, ld=None, ldz=None):
    """dstats bits [R][2L]: dmu = bf16_rn(RN(g + RN(ks mu))), dlv = bf16_rn(RN(RN(RN(RN(0.5 g) eps) E(RN(0.5 lv))) +
    RN(RN(ks 0.5) RN(E(lv) - 1)))), g = float(dz), ks = kl_scale"""
    ld = 2 * L if ld is None else ld
    ldz = L if ldz is None else ldz
    mu, lv = _stats(stats_bits, R, L, ld)
    g = bits_f32(np.asarray(dz_bits, np.uint16).reshape(-1)[:R * ldz].reshape(R, ldz)[:, :L])
    ks = F32(kl_scale)
    with np.errstate(all="ignore"):
        dmu = g + ks * mu
        a = ((F32(0.5) * g) * eps(R, L, seed, call)) * exp_f32(F32(0.5) * lv)
        dlv = a + (ks * F32(0.5)) * (exp_f32(lv) - F32(1))
    return np.concatenate([bf16_bits(dmu), bf16_bits(dlv)], 1)


def bce_replay(logit_bits, target_bits, C, scale, target_stride=None):
    """(dlogits bits [pixels][C], loss float32 [pixels]) of pcnn_bce_logits_bf16: x = float(logit), t = float(target); e =
    E(-|x|); term = RN(RN(max(x, 0) - RN(x t)) + log1p_f32(e)); sigma = RN((x >= 0 ? 1 : e) / RN(1 + e)); dlogits =
    bf16_rn(RN(scale RN(sigma - t))); loss the fp32 sum from +0 of the terms in ascending c"""
    ts = C if target_stride is None else target_stride
    x = bits_f32(logit_bits).reshape(-1, C)
    t = bits_f32(target_bits).reshape(-1, ts)[:, :C]
    with np.errstate(all="ignore"):
        e = exp_f32(-np.abs(x))
        mx = np.where(x > 0, x, F32(0)).astype(F32)                       # max(x, 0) as x > 0 ? x : +0 (a NaN x: x t is NaN)
        term = (mx - x * t) + log1p_f32(e)
        sig = np.where(x >= 0, F32(1), e).astype(F32) / (F32(1) + e)
        g = F32(scale) * (sig - t)
        loss = np.zeros(x.shape[0], F32)
        for c in range(C):
            loss = loss + term[:, c]
    return bf16_bits(g), loss.astype(F32)
