"""numpy reference of the NHWC max pool (pcnn_maxpool_nhwc_bf16_fwd / _bwd, include/pcnn.h), on arrays [N][H][W][C].

Forward: over the in-image positions of a window, r then s, a position is taken when it is the first one, when its value is
greater than the maximum so far, or when it is NaN (first maximum wins, last NaN wins).  Backward: dx sums dy over the windows
whose argmax points at an element, in ascending p then q, starting from the first term; the bf16 form rounds the float32 sum
once, keeps dy's bits when there is one term and gives +0 when there is none."""
import numpy as np


def out_size(H, W, R, S, stride, pad_h, pad_w):
    return (H + 2 * pad_h - R) // stride + 1, (W + 2 * pad_w - S) // stride + 1


def _windows(H, W, R, S, stride, pad_h, pad_w):
    """for every tap (r, s) in scan order: the image rows / columns it reads for every output row / column and their validity"""
    P, Q = out_size(H, W, R, S, stride, pad_h, pad_w)
    for r in range(R):
        h = np.arange(P) * stride - pad_h + r
        for s in range(S):
            w = np.arange(Q) * stride - pad_w + s
            yield r, s, h, w, (h >= 0) & (h < H), (w >= 0) & (w < W)


def fwd_argmax(x, R, S, stride, pad_h, pad_w):
    """argmax bytes r*S + s [N][P][Q][C] (int64) of x (any float dtype: the comparisons are exact)"""
    N, H, W, C = x.shape
    P, Q = out_size(H, W, R, S, stride, pad_h, pad_w)
    m = np.full((N, P, Q, C), -np.inf, x.dtype)
    a = np.full((N, P, Q, C), -1, np.int64)
    for r, s, h, w, vh, vw in _windows(H, W, R, S, stride, pad_h, pad_w):
        v = x[:, np.clip(h, 0, H - 1)][:, :, np.clip(w, 0, W - 1)]
        valid = (vh[:, None] & vw[None, :])[None, :, :, None]
        with np.errstate(invalid="ignore"):
            take = valid & ((a < 0) | (v > m) | np.isnan(v))
        m = np.where(take, v, m)
        a = np.where(take, r * S + s, a)
    assert (a >= 0).all()
    return a


def winner_hw(a, S, stride, pad_h, pad_w):
    """image row and column of each argmax"""
    _, P, Q, _ = a.shape
    h = np.arange(P)[None, :, None, None] * stride - pad_h + a // S
    w = np.arange(Q)[None, None, :, None] * stride - pad_w + a % S
    return h, w


def gather(x, a, S, stride, pad_h, pad_w):
    """x at the argmax of every window: y (the bits of x when x is a bit pattern array)"""
    h, w = winner_hw(a, S, stride, pad_h, pad_w)
    n = np.arange(x.shape[0])[:, None, None, None]
    c = np.arange(x.shape[3])[None, None, None, :]
    return x[n, h, w, c]


def bwd_sum(dy, a, H, W, R, S, stride, pad_h, pad_w):
    """dx [N][H][W][C] in dy's dtype and the number of terms of each element.  Terms in ascending (p, q) are taps in descending
    (r, s); one tap maps distinct windows to distinct elements, so each tap is one vectorised update."""
    N, P, Q, C = dy.shape
    acc = np.zeros((N, H, W, C), dy.dtype)
    cnt = np.zeros((N, H, W, C), np.int64)
    for r in range(R - 1, -1, -1):
        h = np.arange(P) * stride - pad_h + r
        vp = np.nonzero((h >= 0) & (h < H))[0]
        for s in range(S - 1, -1, -1):
            w = np.arange(Q) * stride - pad_w + s
            vq = np.nonzero((w >= 0) & (w < W))[0]
            if vp.size == 0 or vq.size == 0:
                continue
            sel = a[:, vp][:, :, vq] == r * S + s
            d = dy[:, vp][:, :, vq]
            hi, wi = h[vp][:, None], w[vq][None, :]
            old, n0 = acc[:, hi, wi, :], cnt[:, hi, wi, :]
            with np.errstate(invalid="ignore", over="ignore"):
                acc[:, hi, wi, :] = np.where(sel, np.where(n0 > 0, old + d, d), old)
            cnt[:, hi, wi, :] = n0 + sel
    return acc, cnt


def bwd_bf16(pkg, dy_bits, a, H, W, R, S, stride, pad_h, pad_w):
    """dx bits of pcnn_maxpool_nhwc_bf16_bwd: the float32 sum rounded once; dy's bits for one term; +0 for none"""
    acc, cnt = bwd_sum(pkg.bf16_bits_to_f32(dy_bits), a, H, W, R, S, stride, pad_h, pad_w)
    one, _ = bwd_sum(dy_bits.astype(np.int64), a, H, W, R, S, stride, pad_h, pad_w)
    return np.where(cnt == 0, 0, np.where(cnt == 1, one, pkg.f32_to_bf16_bits(acc))).astype(np.uint16)
