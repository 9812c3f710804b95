"""numpy replays of the grouped convolution (pcnn_gconv_plan_create / pcnn_conv_tc_fwd, pcnn_gconv_dgrad, pcnn_gconv_wgrad;
include/pcnn.h) on arrays x [N][H][W][C], w [K][R][S][Cg], dy [N][P][Q][K] with G groups, and float64 references for all three
passes.

In float32 every operation below is the kernels' own, in their order: a product of two bf16 values is exact in float32, so
numpy's rounded product followed by a rounded add gives the bits of the kernels' FMA.  A sum starts from -0, which is the same as
starting from the first term (-0 + v is v for every v, -0 and NaN included).  Taps outside the image read x = +0 and are
multiplied like any other, so 0 * Inf gives NaN.  Output k belongs to group k // Kg, input channel c to group c // Cg."""
import numpy as np

from dwconv_ref import _padded, out_size  # noqa: F401  (the window arithmetic is the depthwise one)


def fwd(x, w, G, b=None, stride=1, pad_h=0, pad_w=0, act=0):
    """y [N][P][Q][K] in x's dtype: the sum over r, then s, then c of x * w from the first term, + b, then act (3: v < 0 ? +0 : v)"""
    N, H, W, C = x.shape
    K, R, S, Cg = w.shape
    Kg = K // G
    P, Q = out_size(H, W, R, S, stride, pad_h, pad_w)
    xp = _padded(x, pad_h, pad_w)
    base = (np.arange(K) // Kg) * Cg                                   # first input channel of each output's group
    acc = np.full((N, P, Q, K), -0.0, x.dtype)
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(R):
            for s in range(S):
                v = xp[:, r:r + (P - 1) * stride + 1:stride, s:s + (Q - 1) * stride + 1:stride]
                for c in range(Cg):
                    acc = acc + v[..., base + c] * w[:, r, s, c].astype(x.dtype)
        if b is not None:
            acc = acc + b.astype(x.dtype)
        if act == 3:
            acc = np.where(acc < 0, np.zeros((), x.dtype), acc)
    return acc


def dgrad(dy, w, G, H, W, stride=1, pad_h=0, pad_w=0):
    """dx [N][H][W][C] in dy's dtype: the sum of dy * w over the taps that reach each element, in ascending r, then s, then k of the
    group, from the first term; +0 with no term.  One tap maps distinct windows to distinct elements, so a tap adds at most once to
    each.  Also returns the number of taps reaching each (h, w)."""
    N, P, Q, K = dy.shape
    _, R, S, Cg = w.shape
    Kg, C = K // G, Cg * G
    cs = np.arange(C)
    kbase, cl = (cs // Cg) * Kg, cs % Cg                               # first output of each input channel's group, its index there
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
                d = dy[:, vp][:, :, vq]
                cur = acc[:, hi, wi, :]
                for k in range(Kg):
                    cur = cur + d[..., kbase + k] * w[kbase + k, r, s, cl].astype(dy.dtype)
                acc[:, hi, wi, :] = cur
                terms[hi, wi] += 1
    return np.where((terms == 0)[None, :, :, None], np.zeros((), dy.dtype), acc), terms


def wgrad_f64(x, dy, G, R, S, stride=1, pad_h=0, pad_w=0):
    """dw [K][R][S][Cg] in float64: the sum over n, p, q of dy[k] * x[group's channel c] (x +0 outside the image)"""
    N, P, Q, K = dy.shape
    C = x.shape[3]
    Kg, Cg = K // G, C // G
    xp = _padded(x.astype(np.float64), pad_h, pad_w)
    d = dy.astype(np.float64).reshape(N, P, Q, G, Kg)
    dw = np.zeros((K, R, S, Cg))
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(R):
            for s in range(S):
                v = xp[:, r:r + (P - 1) * stride + 1:stride, s:s + (Q - 1) * stride + 1:stride].reshape(N, P, Q, G, Cg)
                dw[:, r, s, :] = np.einsum("npqgk,npqgc->gkc", d, v).reshape(K, Cg)
    return dw


def wgrad_abs_f64(x, dy, G, R, S, stride=1, pad_h=0, pad_w=0):
    """the sum of |dy * x| behind each dw[k][r][s][c] (the scale of its error bound)"""
    return wgrad_f64(np.abs(x), np.abs(dy), G, R, S, stride, pad_h, pad_w)


def fwd_f64(x, w, G, b=None, stride=1, pad_h=0, pad_w=0, act=0):
    return fwd(x.astype(np.float64), w.astype(np.float64), G, None if b is None else b.astype(np.float64), stride, pad_h, pad_w, act)


def dgrad_f64(dy, w, G, H, W, stride=1, pad_h=0, pad_w=0):
    return dgrad(dy.astype(np.float64), w.astype(np.float64), G, H, W, stride, pad_h, pad_w)[0]
