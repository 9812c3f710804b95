"""numpy replays of the NHWC average pools (pcnn_avgpool_nhwc_bf16_fwd / _bwd, pcnn_global_avgpool_nhwc_bf16_fwd / _bwd,
include/pcnn.h) on arrays [N][H][W][C], and float64 references.

In float32 every operation below is the kernels' own, in their order: numpy adds and divides float32 arrays with one IEEE
rounding each.  A sum starts from -0, which is the same as starting from the first term (-0 + v is v for every v, -0 and NaN
included)."""
import numpy as np

from maxpool_ref import out_size

U = 2.0 ** -24


def counts(H, W, R, S, stride, pad_h, pad_w, count_include_pad):
    """cnt[p][q]: R*S, or the window's in-image positions"""
    P, Q = out_size(H, W, R, S, stride, pad_h, pad_w)
    if count_include_pad:
        return np.full((P, Q), R * S, np.int64)
    h0, w0 = np.arange(P) * stride - pad_h, np.arange(Q) * stride - pad_w
    rows = np.minimum(R, H - h0) - np.maximum(0, -h0)
    cols = np.minimum(S, W - w0) - np.maximum(0, -w0)
    return rows[:, None] * cols[None, :]


def fwd(x, R, S, stride, pad_h, pad_w, count_include_pad):
    """y [N][P][Q][C] in x's dtype: the in-image sum of each window, r then s, over cnt"""
    N, H, W, C = x.shape
    P, Q = out_size(H, W, R, S, stride, pad_h, pad_w)
    acc = np.full((N, P, Q, C), -0.0, x.dtype)
    for r in range(R):
        h = np.arange(P) * stride - pad_h + r
        for s in range(S):
            w = np.arange(Q) * stride - pad_w + s
            v = x[:, np.clip(h, 0, H - 1)][:, :, np.clip(w, 0, W - 1)]
            valid = (((h >= 0) & (h < H))[:, None] & ((w >= 0) & (w < W))[None, :])[None, :, :, None]
            with np.errstate(invalid="ignore", over="ignore"):
                acc = np.where(valid, acc + v, acc)
    cnt = counts(H, W, R, S, stride, pad_h, pad_w, count_include_pad).astype(x.dtype)[None, :, :, None]
    with np.errstate(invalid="ignore", over="ignore"):
        return acc / cnt


def bwd(dy, H, W, R, S, stride, pad_h, pad_w, count_include_pad):
    """dx [N][H][W][C] in dy's dtype: the sum of dy / cnt over the windows containing each element in ascending (p, q), +0 with no
    term.  Terms in ascending (p, q) are taps in descending (r, s); one tap maps distinct windows to distinct elements."""
    N, P, Q, C = dy.shape
    cnt = counts(H, W, R, S, stride, pad_h, pad_w, count_include_pad).astype(dy.dtype)[None, :, :, None]
    with np.errstate(invalid="ignore", over="ignore"):
        t = dy / cnt
    acc = np.full((N, H, W, C), -0.0, dy.dtype)
    terms = np.zeros((H, W), np.int64)
    for r in range(R - 1, -1, -1):
        h = np.arange(P) * stride - pad_h + r
        vp = np.nonzero((h >= 0) & (h < H))[0]
        for s in range(S - 1, -1, -1):
            w = np.arange(Q) * stride - pad_w + s
            vq = np.nonzero((w >= 0) & (w < W))[0]
            if vp.size == 0 or vq.size == 0:
                continue
            hi, wi = h[vp][:, None], w[vq][None, :]
            with np.errstate(invalid="ignore", over="ignore"):
                acc[:, hi, wi, :] = acc[:, hi, wi, :] + t[:, vp][:, :, vq]
            terms[hi, wi] += 1
    return np.where((terms == 0)[None, :, :, None], np.zeros((), dy.dtype), acc), terms


def global_fwd(x, info):
    """y [N][C] in x's dtype, summed in the order of the partition `info` (global_avgpool_nhwc_info): in each range of
    pixels_per_cta pixels, lane l sums the pixels l, l + lanes, ...; the lanes holding a pixel are added in lane order, then the
    ranges in range order; then / H*W"""
    N, H, W, C = x.shape
    HW = H * W
    xs = x.reshape(N, HW, C)
    lanes, per = info["lanes"], info["pixels_per_cta"]
    assert info["ranges"] == -(-HW // per)
    total = np.full((N, C), -0.0, x.dtype)
    with np.errstate(invalid="ignore", over="ignore"):
        for p0 in range(0, HW, per):
            acc = np.full((N, lanes, C), -0.0, x.dtype)
            for j in range(per // lanes):
                px = p0 + j * lanes + np.arange(lanes)
                ok = px < HW
                acc[:, ok] = acc[:, ok] + xs[:, px[ok]]
            s = np.full((N, C), -0.0, x.dtype)
            for lane in range(min(lanes, HW - p0)):
                s = s + acc[:, lane]
            total = total + s
        return total / x.dtype.type(HW)


def global_f64(x):
    """the float64 mean over the pixels of each image and channel: [N][C]"""
    return x.astype(np.float64).mean(axis=(1, 2))


def gap_bound(pkg, xf, info):
    """[lo, hi] of the error model of the global pool's y (test_avgpool_nhwc_gpu.py's docstring) for every y, as float32 values:
    returns the float64 mean m, the bound E of |fp32 sum / (H*W) - m|, and m - E and m + E rounded to bf16"""
    N, H, W, C = xf.shape
    n_acc = (info["pixels_per_cta"] // info["lanes"] - 1) + (info["lanes"] - 1) + (info["ranges"] - 1)
    gamma = n_acc * U / (1 - n_acc * U)
    x64 = xf.astype(np.float64)
    S, A = x64.sum(axis=(1, 2)), np.abs(x64).sum(axis=(1, 2))
    m, E = S / (H * W), (gamma * A + U * (np.abs(S) + gamma * A)) / (H * W)
    bf, f32 = pkg.f32_to_bf16_bits, pkg.bf16_bits_to_f32
    return m, E, f32(bf((m - E).astype(np.float32))), f32(bf((m + E).astype(np.float32)))


def global_bwd(dy, H, W):
    """dx [N][H][W][C] = dy / H*W at every pixel, in dy's dtype"""
    q = dy / dy.dtype.type(H * W)
    return np.broadcast_to(q[:, None, None, :], (dy.shape[0], H, W, dy.shape[1]))
