"""Float64 reference of self-attention (pcnn_attention_bf16_fwd / _bwd), the error bounds the device is held to, and a float32 /
bf16 emulation of the rounding points include/pcnn.h states, which the CPU tests keep inside those bounds.  The emulation rounds
where the device rounds (u, u - m, P, l, acc, 1 / l, O, lse, D, dS and the outputs), but it sums in numpy's float32 order, not
the device's per-thread sums and shuffles, and it takes exactly rounded exp2 for ex2.approx.  So it checks that the bounds cover
the stated roundings in one summation order; the error terms below carry the summation order (T 2^-24) and ex2.approx (2^-22)
separately, and the device itself is held to the bounds against float64 by tests/test_attention_gpu.py.

Arrays are [N][T][h][d] (tokens in NHWC pixel order, head j at columns j d), lse is [N][h][T].

Error model, per output element, with the reference's P = softmax(scale S) and every input already bf16 (both sides read the same
values).  u = 2^-8:
  * O[t]   : 2 u sum_j P[t, j] |v[j]| + u |O[t]|.  P rounded to bf16 moves each term by at most 2^-9 relative, and l, the sum of
             those bf16 values, by at most 2^-9: together 2^-8 of sum P |v|.  The fp32 score u = RN(s c2), RN(u - m), ex2.approx
             and the fp32 sums over T <= 16384 terms add at most T 2^-24 + 2^-21 relative at logits |scale s| <= 2^7, and 2^-10
             at |scale s| <= 10^4 with exact products: the second 2^-8 of c = 2 covers them.  The last u |O| is the bf16 output.
  * lse[t] : 2^-7 + 2^-20 |lse|.  l is within 2^-9 relative of sum exp, lg2.approx adds 2^-21, and m, m + lg2(l) and the ln 2
             product are three fp32 roundings of a value of size |lse| (2^-22 |lse| each with margin).
  * dV[j]  : 2 u sum_t P[t, j] |dO[t]| + u |dV[j]|: bf16 P as in O, the fp32 sum, the bf16 output.
  * dQ[t]  : 2 u scale sum_j P[t, j] (|dP[t, j]| + Dabs[t]) |k[j]| + u |dQ[t]|, Dabs[t] = sum_i |dO[t, i]| |O[t, i]|.
             dS = P (dP - D) carries 2^-9 from the recomputed P (ex2 of RN(RN(s c2) - RN(lse log2 e)), within 2^-10 at large
             logits) and 2^-9 from its bf16 rounding.  D is formed from the bf16 O, 2^-9 relative per term, so its error is
             2^-9 Dabs, not 2^-9 |D|: D is a sum of signed terms that may cancel.  That error is common to every key of the row
             and does not cancel in sum_j dS k (keys tied at the maximum share one k), so it enters with weight P |k|.  dP - D
             in fp32 adds d 2^-24 (|dP| + Dabs).
  * dK[j]  : 2 u scale sum_t P[t, j] (|dP[t, j]| + Dabs[t]) |q[t]| + u |dK[j]|, as dQ.
Every bound also carries an absolute TINY = 2^-100: ex2.approx flushes a P below 2^-126 to zero, which moves an output of inputs up
to 2^20 in size by less than that.
"""
import numpy as np

U = 2.0 ** -8
TINY = 2.0 ** -100
LOG2E = 1.4426950408889634
LN2 = 0.6931471805599453


def bf16(a):
    """round float32 to bf16 (nearest even), returned as float32; NaN stays NaN"""
    a = np.ascontiguousarray(a, np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    out = r.astype(np.uint32).view(np.float32)
    return np.where(np.isnan(a), np.float32(np.nan), out).astype(np.float32)


def _heads(a):
    return np.transpose(np.asarray(a, np.float64), (0, 2, 1, 3))          # [N][h][T][d]


def _tokens(a):
    return np.transpose(a, (0, 2, 1, 3))                                   # back to [N][T][h][d]


def forward(q, k, v, scale):
    """float64 O [N][T][h][d], lse [N][h][T] and P [N][h][T][T]"""
    qh, kh, vh = _heads(q), _heads(k), _heads(v)
    s = (qh @ np.swapaxes(kh, -1, -2)) * scale
    m = s.max(-1, keepdims=True)
    e = np.exp(s - m)
    den = e.sum(-1, keepdims=True)
    p = e / den
    return _tokens(p @ vh), (m + np.log(den))[..., 0], p


def backward(q, k, v, dout, scale):
    """float64 dq, dk, dv [N][T][h][d], with P, dP and D [N][h][T] for the bounds"""
    qh, kh, vh, dh = _heads(q), _heads(k), _heads(v), _heads(dout)
    o, lse, p = forward(q, k, v, scale)
    dv = np.swapaxes(p, -1, -2) @ dh
    dp = dh @ np.swapaxes(vh, -1, -2)
    D = np.sum(dh * _heads(o), -1)
    ds = p * (dp - D[..., None])
    dq = (ds @ kh) * scale
    dk = (np.swapaxes(ds, -1, -2) @ qh) * scale
    return _tokens(dq), _tokens(dk), _tokens(dv), p, dp, D


def bounds(q, k, v, dout, scale):
    """{name: (reference, bound)} for o, lse, dq, dk and dv, in the form of the module docstring"""
    qh, kh, vh, dh = _heads(q), _heads(k), _heads(v), _heads(dout)
    o, lse, p = forward(q, k, v, scale)
    dq, dk, dv, _, dp, D = backward(q, k, v, dout, scale)
    pt = np.swapaxes(p, -1, -2)
    bo = 2 * U * _tokens(p @ np.abs(vh)) + U * np.abs(o)
    blse = 2 * U + 2.0 ** -20 * np.abs(lse)
    bdv = 2 * U * _tokens(pt @ np.abs(dh)) + U * np.abs(dv)
    dabs = np.sum(np.abs(dh) * np.abs(_heads(o)), -1)                    # sum |dO| |O|: what D's rounding errors are relative to
    w = p * (np.abs(dp) + dabs[..., None])
    bdq = 2 * U * scale * _tokens(w @ np.abs(kh)) + U * np.abs(dq)
    bdk = 2 * U * scale * _tokens(np.swapaxes(w, -1, -2) @ np.abs(qh)) + U * np.abs(dk)
    return dict(o=(o, bo + TINY), lse=(lse, blse), dq=(dq, bdq + TINY), dk=(dk, bdk + TINY), dv=(dv, bdv + TINY))


def worst(got, ref, bound):
    """largest |got - ref| / bound (NaN where got is not finite counts as infinite)"""
    got = np.asarray(got, np.float64)
    err = np.where(np.isfinite(got), np.abs(got - ref), np.inf)
    ratio = np.divide(err, bound, out=np.where(err > 0, np.inf, 0.0), where=bound > 0)    # an exact 0 needs no bound
    return float(np.max(ratio))


def _ex2(x):
    return np.exp2(x.astype(np.float64)).astype(np.float32)


def emulate(q, k, v, dout, scale, block=64):
    """The stated operation order in float32 with the stated bf16 roundings (one key block of 64 at a time), on bf16 inputs:
    returns o, lse, dq, dk, dv as float32 (o, dq, dk and dv rounded to bf16)."""
    q, k, v, dout = (np.asarray(a, np.float32) for a in (q, k, v, dout))
    N, T, h, d = q.shape
    f = np.float32
    c2 = f(scale * LOG2E)
    qh, kh, vh, dh = (np.transpose(a, (0, 2, 1, 3)) for a in (q, k, v, dout))     # [N][h][T][d]
    s_all = np.einsum("nhti,nhsi->nhts", qh, kh, dtype=np.float32)
    m = np.full((N, h, T), -np.inf, f)
    l = np.zeros((N, h, T), f)
    acc = np.zeros((N, h, T, d), f)
    for b0 in range(0, T, block):
        u = (s_all[..., b0:b0 + block] * c2).astype(f)
        mn = np.maximum(m, u.max(-1))
        alpha = _ex2((m - mn).astype(f))
        P = bf16(_ex2((u - mn[..., None]).astype(f)))
        l = (l * alpha + P.sum(-1, dtype=np.float32)).astype(f)
        acc = (acc * alpha[..., None] + np.einsum("nhts,nhsi->nhti", P, vh[:, :, b0:b0 + block], dtype=np.float32)).astype(f)
        m = mn
    o = bf16(acc * (f(1) / l)[..., None])
    lse = ((m + np.log2(l.astype(np.float64)).astype(f)) * f(LN2)).astype(f)
    D = np.einsum("nhti,nhti->nht", dh, o, dtype=np.float32)
    l2 = (lse * f(LOG2E)).astype(f)
    P = _ex2(((s_all * c2).astype(f) - l2[..., None]).astype(f))
    dp = np.einsum("nhti,nhsi->nhts", dh, vh, dtype=np.float32)
    ds = bf16(P * (dp - D[..., None]).astype(f))
    dv = bf16(np.einsum("nhts,nhti->nhsi", bf16(P), dh, dtype=np.float32))
    dq = bf16(np.einsum("nhts,nhsi->nhti", ds, kh, dtype=np.float32) * f(scale))
    dk = bf16(np.einsum("nhts,nhti->nhsi", ds, qh, dtype=np.float32) * f(scale))
    back = lambda a: np.transpose(a, (0, 2, 1, 3))
    return back(o), lse, back(dq), back(dk), back(dv)
