"""numpy replays of the depthwise convolution (pcnn_dwconv_plan_create / pcnn_conv_tc_fwd, pcnn_dwconv_dgrad, pcnn_dwconv_wgrad;
include/pcnn.h) on arrays x [N][H][W][C], w [C][R][S], dy [N][P][Q][C], and float64 references for all three passes.

In float32 every operation below is the kernels' own, in their order: a product of two bf16 values is exact in float32, so
numpy's rounded product followed by a rounded add gives the bits of the kernels' FMA.  A sum starts from -0, which is the same as
starting from the first term (-0 + v is v for every v, -0 and NaN included).  Taps outside the image read x = +0 and are
multiplied like any other, so 0 * Inf gives NaN."""
import numpy as np


def out_size(H, W, R, S, stride, pad_h, pad_w):
    return (H + 2 * pad_h - R) // stride + 1, (W + 2 * pad_w - S) // stride + 1


def _padded(x, pad_h, pad_w, extra_h=0, extra_w=0):
    """x with pad_h / pad_w rows and columns of +0 around it (and extra ones at the far edges, never read by a valid window)"""
    N, H, W, C = x.shape
    xp = np.zeros((N, H + 2 * pad_h + extra_h, W + 2 * pad_w + extra_w, C), x.dtype)
    xp[:, pad_h:pad_h + H, pad_w:pad_w + W] = x
    return xp


def fwd(x, w, b=None, stride=1, pad_h=0, pad_w=0, act=0):
    """y [N][P][Q][C] in x's dtype: the sum over r, then s, of x * w from the first term, + b, then act (3: v < 0 ? +0 : v)"""
    N, H, W, C = x.shape
    _, R, S = w.shape
    P, Q = out_size(H, W, R, S, stride, pad_h, pad_w)
    xp = _padded(x, pad_h, pad_w)
    acc = np.full((N, P, Q, C), -0.0, x.dtype)
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(R):
            for s in range(S):
                v = xp[:, r:r + (P - 1) * stride + 1:stride, s:s + (Q - 1) * stride + 1:stride]
                acc = acc + v * w[:, r, s].astype(x.dtype)
        if b is not None:
            acc = acc + b.astype(x.dtype)
        if act == 3:
            acc = np.where(acc < 0, np.zeros((), x.dtype), acc)
    return acc


def dgrad(dy, w, H, W, stride=1, pad_h=0, pad_w=0):
    """dx [N][H][W][C] in dy's dtype: the sum of dy * w over the taps that reach each element, in ascending r, then s, from the
    first term; +0 with no term.  One tap maps distinct windows to distinct elements, so a tap adds at most once to each."""
    N, P, Q, C = dy.shape
    _, R, S = w.shape
    acc = np.full((N, H, W, C), -0.0, dy.dtype)
    terms = np.zeros((H, W), np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(R):
            h = np.arange(P) * stride - pad_h + r
            vp = np.nonzero((h >= 0) & (h < H))[0]
            for s in range(S):
                ww = np.arange(Q) * stride - pad_w + s
                vq = np.nonzero((ww >= 0) & (ww < W))[0]
                if vp.size == 0 or vq.size == 0:
                    continue
                hi, wi = h[vp][:, None], ww[vq][None, :]
                acc[:, hi, wi, :] = acc[:, hi, wi, :] + dy[:, vp][:, :, vq] * w[:, r, s].astype(dy.dtype)
                terms[hi, wi] += 1
    return np.where((terms == 0)[None, :, :, None], np.zeros((), dy.dtype), acc), terms


def wgrad_f64(x, dy, R, S, stride=1, pad_h=0, pad_w=0):
    """dw [C][R][S] in float64: the sum over n, p, q of dy * x (x +0 outside the image)"""
    N, P, Q, C = dy.shape
    xp = _padded(x.astype(np.float64), pad_h, pad_w)
    d = dy.astype(np.float64)
    dw = np.zeros((C, R, S))
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(R):
            for s in range(S):
                v = xp[:, r:r + (P - 1) * stride + 1:stride, s:s + (Q - 1) * stride + 1:stride]
                dw[:, r, s] = np.einsum("npqc,npqc->c", d, v)
    return dw


def wgrad_abs_f64(x, dy, R, S, stride=1, pad_h=0, pad_w=0):
    """the sum of |dy * x| behind each dw[c][r][s] (the scale of its error bound)"""
    return wgrad_f64(np.abs(x), np.abs(dy), R, S, stride, pad_h, pad_w)


def fwd_f64(x, w, b=None, stride=1, pad_h=0, pad_w=0, act=0):
    return fwd(x.astype(np.float64), w.astype(np.float64), None if b is None else b.astype(np.float64), stride, pad_h, pad_w, act)


def dgrad_f64(dy, w, H, W, stride=1, pad_h=0, pad_w=0):
    return dgrad(dy.astype(np.float64), w.astype(np.float64), H, W, stride, pad_h, pad_w)[0]
