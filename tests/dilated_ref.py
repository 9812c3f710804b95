"""References for dilated ("atrous") convolution (pcnn_conv_wide_*_dilated, pcnn_dwconv_plan_create_dilated; include/pcnn.h).

Tap (r, s) of output (p, q) reads x~[p*stride - pad_h + r*dil_h][q*stride - pad_w + s*dil_w], x~ = +0 outside the image, with
    P = (H + 2 pad_h - dil_h (R - 1) - 1) // stride + 1,   Q = (W + 2 pad_w - dil_w (S - 1) - 1) // stride + 1.

* Wide (NHWC x, KRSC f [K][R][S][C], dy [N][P][Q][K]): float64 forward, weight gradient and input gradient, written from the
  formulas by slicing a zero-padded canvas.  The input gradient scatters each tap's products into the canvas and crops it.
* Depthwise (x [N][H][W][C], w [C][R][S]): float32 replays of the forward and the input gradient in the kernels' order (ascending
  r, then s, from the first term; a product of two bf16 values is exact in float32, so a rounded product and a rounded add give the
  bits of the kernels' FMA), and a float64 weight gradient.  At dilation 1 these are dwconv_ref's."""
import numpy as np


def out_size(H, W, R, S, stride=1, padding=(0, 0), dilation=(1, 1)):
    (ph, pw), (dh, dw) = padding, dilation
    return (H + 2 * ph - dh * (R - 1) - 1) // stride + 1, (W + 2 * pw - dw * (S - 1) - 1) // stride + 1


def _canvas(x, ph, pw, dtype=np.float64):
    N, H, W, C = x.shape
    xp = np.zeros((N, H + 2 * ph, W + 2 * pw, C), dtype)
    xp[:, ph:ph + H, pw:pw + W] = x
    return xp


def _tap(xp, r, s, P, Q, stride, dilation):
    """the [N][P][Q][C] view of the canvas that tap (r, s) reads"""
    h0, w0 = r * dilation[0], s * dilation[1]
    return xp[:, h0:h0 + (P - 1) * stride + 1:stride, w0:w0 + (Q - 1) * stride + 1:stride]


# ------------------------------------------------------------------------------------------------------------- wide, float64
def fwd_f64(x, f, b=None, stride=1, padding=(0, 0), dilation=(1, 1)):
    """y [N][P][Q][K] = b + sum_{r,s,c} x~ * f (no activation)"""
    N, H, W, C = x.shape
    K, R, S, _ = f.shape
    P, Q = out_size(H, W, R, S, stride, padding, dilation)
    xp = _canvas(np.asarray(x, np.float64), *padding)
    f = np.asarray(f, np.float64)
    y = np.zeros((N, P, Q, K))
    for r in range(R):
        for s in range(S):
            y += _tap(xp, r, s, P, Q, stride, dilation) @ f[:, r, s, :].T
    if b is not None:
        y += np.asarray(b, np.float64)
    return y


def wgrad_f64(x, dy, R, S, stride=1, padding=(0, 0), dilation=(1, 1)):
    """dw [K][R][S][C] = sum_{n,p,q} dy * x~"""
    N, P, Q, K = dy.shape
    C = x.shape[3]
    xp = _canvas(np.asarray(x, np.float64), *padding)
    d = np.asarray(dy, np.float64)
    dw = np.zeros((K, R, S, C))
    for r in range(R):
        for s in range(S):
            dw[:, r, s, :] = d.reshape(-1, K).T @ np.ascontiguousarray(_tap(xp, r, s, P, Q, stride, dilation)).reshape(-1, C)
    return dw


def dgrad_f64(dy, f, H, W, stride=1, padding=(0, 0), dilation=(1, 1)):
    """dx [N][H][W][C] = sum_{k,r,s} dy * f over the taps that reach each element"""
    N, P, Q, K = dy.shape
    _, R, S, C = f.shape
    ph, pw = padding
    d, f = np.asarray(dy, np.float64), np.asarray(f, np.float64)
    canvas = np.zeros((N, H + 2 * ph, W + 2 * pw, C))
    for r in range(R):
        for s in range(S):
            _tap(canvas, r, s, P, Q, stride, dilation)[...] += d @ f[:, r, s, :]
    return canvas[:, ph:ph + H, pw:pw + W]


def zero_inserted(f, dilation):
    """the filters [K][R][S][C] spread to the dense E_h x E_w window, zeros between the taps: the undilated convolution with these
    filters is the dilated one"""
    K, R, S, C = f.shape
    dh, dw = dilation
    out = np.zeros((K, dh * (R - 1) + 1, dw * (S - 1) + 1, C), f.dtype)
    out[:, ::dh, ::dw, :] = f
    return out


# ------------------------------------------------------------------------------------------------------------------- depthwise
def dw_fwd(x, w, b=None, stride=1, padding=(0, 0), dilation=(1, 1), act=0):
    """y [N][P][Q][C] in x's dtype: the sum over r, then s, of x~ * w from the first term, + b, then act (3: v < 0 ? +0 : v)"""
    N, H, W, C = x.shape
    _, R, S = w.shape
    P, Q = out_size(H, W, R, S, stride, padding, dilation)
    xp = _canvas(x, *padding, dtype=x.dtype)
    acc = np.full((N, P, Q, C), -0.0, x.dtype)
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(R):
            for s in range(S):
                acc = acc + _tap(xp, r, s, P, Q, stride, dilation) * w[:, r, s].astype(x.dtype)
        if b is not None:
            acc = acc + b.astype(x.dtype)
        if act == 3:
            acc = np.where(acc < 0, np.zeros((), x.dtype), acc)
    return acc


def dw_dgrad(dy, w, H, W, stride=1, padding=(0, 0), dilation=(1, 1)):
    """dx [N][H][W][C] in dy's dtype: the sum of dy * w over the taps that reach each element, in ascending r, then s, from the
    first term; +0 with no term.  A tap maps distinct windows to distinct elements, so it adds at most once to each."""
    N, P, Q, C = dy.shape
    _, R, S = w.shape
    (ph, pw), (dh, dw) = padding, dilation
    acc = np.full((N, H, W, C), -0.0, dy.dtype)
    terms = np.zeros((H, W), np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(R):
            h = np.arange(P) * stride - ph + r * dh
            vp = np.nonzero((h >= 0) & (h < H))[0]
            for s in range(S):
                ww = np.arange(Q) * stride - pw + s * dw
                vq = np.nonzero((ww >= 0) & (ww < W))[0]
                if vp.size == 0 or vq.size == 0:
                    continue
                hi, wi = h[vp][:, None], ww[vq][None, :]
                acc[:, hi, wi, :] = acc[:, hi, wi, :] + dy[:, vp][:, :, vq] * w[:, r, s].astype(dy.dtype)
                terms[hi, wi] += 1
    return np.where((terms == 0)[None, :, :, None], np.zeros((), dy.dtype), acc)


def dw_wgrad_f64(x, dy, R, S, stride=1, padding=(0, 0), dilation=(1, 1)):
    """dw [C][R][S] in float64: the sum over n, p, q of dy * x~"""
    N, P, Q, C = dy.shape
    xp = _canvas(np.asarray(x, np.float64), *padding)
    d = np.asarray(dy, np.float64)
    out = np.zeros((C, R, S))
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(R):
            for s in range(S):
                out[:, r, s] = np.einsum("npqc,npqc->c", d, _tap(xp, r, s, P, Q, stride, dilation))
    return out


# ------------------------------------------------------------------------------------------------ the input gradient's phases
def dgrad_phase_taps(a, pad, dil, stride, R):
    """(taps, rho, off, tap step, dy step) of row phase a of dx, as the input-gradient kernel walks it: with g = gcd(dil, stride),
    none unless g | a + pad; then r = rho + (stride/g) i reads dy row u - (dil/g) i + off"""
    g = int(np.gcd(dil, stride))
    tstep, dystep = stride // g, dil // g
    if (a + pad) % g:
        return 0, 0, 0, tstep, dystep
    rho = next(r for r in range(tstep) if (r * dil - a - pad) % stride == 0)
    off = (a + pad - rho * dil) // stride
    taps = -(-(R - rho) // tstep) if rho < R else 0
    return taps, rho, off, tstep, dystep
