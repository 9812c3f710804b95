"""numpy replay of resized batches (pcnn_augment_resized_u8_bf16, include/pcnn.h): the RandomResizedCrop box draws with their
fallback, the Resize + CenterCrop window, torch's uint8 antialiased bilinear resample (PIL-SIMD's fixed point: double weights,
int16 taps, a horizontal pass into uint8, then the vertical pass), and the batch x [N][H_out][W_out][C_out] as bf16 bits.

The permutation, the flip bit and the table are augment_ref's; E is bnact_ref's exp_f32.  numpy float32 and float64 operations
are each one IEEE round to nearest, as the kernel's explicitly rounded ones."""
import math

import numpy as np

import augment_ref as A
from bnact_ref import exp_f32
from dropout_ref import philox4x32_10

TRAIN, EVAL = 1, 2
ATTEMPTS = 10
BOX_DOMAIN = 0xC0000000


# ------------------------------------------------------------------------------------------------ the box
def box_counters(i, k, epoch):
    """the counter words of box block k of images i (uint64 array)"""
    lo, hi = A._words(i)
    return (lo, hi | np.uint64(BOX_DOMAIN | (8 + k) << 24), *A._words(epoch))


def box_constants(scale, ratio):
    """(s0, s range, log r0, log r range) as the host rounds them to fp32"""
    f = np.float32
    s0, s1 = f(scale[0]), f(scale[1])
    l0, l1 = f(math.log(float(f(ratio[0])))), f(math.log(float(f(ratio[1]))))
    return s0, f(s1 - s0), l0, f(l1 - l0)


def uniform(u, low, span):
    """U(u) = RN(RN(RN(float(u >> 8) 2^-24) span) + low) in float32, u uint32 words"""
    x = (np.asarray(u, np.uint64) >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)
    return (x * np.float32(span) + np.float32(low)).astype(np.float32)


def fallback(H, W, ratio):
    """torchvision's central crop when no attempt fits: (top, left, h, w)"""
    in_ratio = float(W) / float(H)
    if in_ratio < min(ratio):
        w, h = W, int(round(W / min(ratio)))
    elif in_ratio > max(ratio):
        h, w = H, int(round(H * max(ratio)))
    else:
        h, w = H, W
    return (H - h) // 2, (W - w) // 2, h, w


def umulhi(word, span):
    return ((np.asarray(word, np.uint64) * np.asarray(span, np.uint64)) >> np.uint64(32)).astype(np.int64)


def choose_box(H, W, s, lr, w_top, w_left, ratio, exp=exp_f32):
    """The box rule on the draws of each image: s, lr float32 [..., 10], w_top / w_left the uint32 words of the randints.  Returns
    (top, left, h, w, attempt) int64 arrays, attempt -1 for the fallback.  exp replaces E (the count of test_resize_cpu)."""
    s, lr = np.asarray(s, np.float32), np.asarray(lr, np.float32)
    shape = s.shape[:-1]
    area = float(H * W)
    h = np.zeros(shape, np.int64)
    w = np.zeros(shape, np.int64)
    attempt = np.full(shape, -1, np.int64)
    for t in range(ATTEMPTS):
        aspect = np.asarray(exp(lr[..., t]), np.float32).astype(np.float64)
        ta = area * s[..., t].astype(np.float64)
        with np.errstate(all="ignore"):
            cw, ch = np.rint(np.sqrt(ta * aspect)), np.rint(np.sqrt(ta / aspect))
        ok = (attempt < 0) & (cw > 0) & (cw <= W) & (ch > 0) & (ch <= H)
        w = np.where(ok, np.nan_to_num(cw).astype(np.int64), w)
        h = np.where(ok, np.nan_to_num(ch).astype(np.int64), h)
        attempt = np.where(ok, t, attempt)
    ft, fl, fh, fw = fallback(H, W, ratio)
    top = np.where(attempt >= 0, umulhi(w_top, np.maximum(H - h + 1, 1)), ft)
    left = np.where(attempt >= 0, umulhi(w_left, np.maximum(W - w + 1, 1)), fl)
    return top, left, np.where(attempt >= 0, h, fh), np.where(attempt >= 0, w, fw), attempt


def box_draws(i, scale, ratio, seed, epoch):
    """(s, lr, w_top, w_left) of images i: s and lr float32 [len(i)][10], the randint words uint32 [len(i)]"""
    i = np.asarray(i, np.uint64)
    s0, sr, l0, lrg = box_constants(scale, ratio)
    blocks = [philox4x32_10(box_counters(i, k, epoch), A._key(seed)) for k in range(ATTEMPTS // 2 + 1)]
    us = np.stack([blocks[t // 2][..., 2 if t & 1 else 0] for t in range(ATTEMPTS)], -1)
    ul = np.stack([blocks[t // 2][..., 3 if t & 1 else 1] for t in range(ATTEMPTS)], -1)
    last = blocks[ATTEMPTS // 2]
    return uniform(us, s0, sr), uniform(ul, l0, lrg), last[..., 0], last[..., 1]


def boxes(i, H, W, scale, ratio, seed, epoch):
    """(top, left, h, w, attempt) of images i in an epoch"""
    s, lr, wt, wl = box_draws(i, scale, ratio, seed, epoch)
    return choose_box(H, W, s, lr, wt, wl, ratio)


# ------------------------------------------------------------------------------------------------ the resample
def axis_weights(n_in, n_out):
    """(xmin, count, q, prec) of an n_in -> n_out axis: first tap and tap count per output, int64 taps q [n_out][taps] at 2^prec
    (0 past the count), and prec"""
    scale = n_in / n_out
    support = scale if scale >= 1.0 else 1.0
    invscale = 1.0 / scale if scale >= 1.0 else 1.0
    taps = int(math.ceil(support)) * 2 + 1
    o = np.arange(n_out, dtype=np.float64)
    center = scale * (o + 0.5)
    xmin = np.maximum(np.trunc(center - support + 0.5).astype(np.int64), 0)
    xmax = np.minimum(np.trunc(center + support + 0.5).astype(np.int64), n_in)
    count = np.clip(xmax - xmin, 0, taps)
    j = np.arange(taps)
    x = np.abs(((j[None, :] + xmin[:, None]).astype(np.float64) - center[:, None] + 0.5) * invscale)
    w = np.where((x < 1.0) & (j[None, :] < count[:, None]), 1.0 - x, 0.0)
    total = np.zeros(n_out)
    for k in range(taps):                                          # the kernel's order
        total = total + w[:, k]
    with np.errstate(invalid="ignore", divide="ignore"):
        w = np.where(total[:, None] != 0.0, w / total[:, None], w)
    wmax = float(w.max()) if w.size else 0.0
    prec = 0
    while prec < 22 and int(0.5 + wmax * (1 << (prec + 1))) < (1 << 15):
        prec += 1
    q = np.trunc(w * float(1 << prec) + 0.5).astype(np.int64)
    return xmin, count, q, prec


def resample_axis(a, axis, n_out):
    """a uint8 array resampled along `axis` to n_out (torch's uint8 antialiased bilinear, one pass)"""
    n_in = a.shape[axis]
    if n_in == n_out:
        return a
    xmin, _, q, prec = axis_weights(n_in, n_out)
    idx = np.minimum(xmin[:, None] + np.arange(q.shape[1])[None, :], n_in - 1)        # taps past the count weigh 0
    t = np.take(a, idx, axis=axis).astype(np.int64)                                    # axis -> (n_out, taps)
    qs = q.reshape((1,) * axis + q.shape + (1,) * (a.ndim - axis - 1))
    acc = (t * qs).sum(axis=axis + 1) + (1 << (prec - 1))
    return np.clip(acc >> prec, 0, 255).astype(np.uint8)


def resample(img, h, w):
    """uint8 [H][W][C] -> [h][w][C]: the horizontal pass, then the vertical"""
    return resample_axis(resample_axis(img, 1, w), 0, h)


# ------------------------------------------------------------------------------------------------ eval geometry
def resized_size(H, W, size):
    """(Rh, Rw): Resize(size) sets the shorter side to size and the longer to int(size long / short)"""
    short, long_ = (W, H) if W <= H else (H, W)
    new_long = int(size * long_ / short)
    return (new_long, size) if W <= H else (size, new_long)


def anchor(R, c):
    """the window's first position on an axis of R pixels for a crop of c (negative: CenterCrop's zero padding)"""
    return -((c - R) // 2) if c > R else int(round((R - c) / 2.0))


def window(img, H_out, W_out, ty, tx):
    """the H_out x W_out window of img at (ty, tx), 0 outside it"""
    R, S = img.shape[:2]
    out = np.zeros((H_out, W_out) + img.shape[2:], np.uint8)
    ys, xs = np.arange(H_out) + ty, np.arange(W_out) + tx
    vy, vx = (ys >= 0) & (ys < R), (xs >= 0) & (xs < S)
    out[np.ix_(vy, vx)] = img[np.ix_(ys[vy], xs[vx])]
    return out


def eval_image(img, resize_size, H_out, W_out):
    """Resize(resize_size) + CenterCrop((H_out, W_out)) of uint8 [H][W][C]"""
    Rh, Rw = resized_size(img.shape[0], img.shape[1], resize_size)
    return window(resample(img, Rh, Rw), H_out, W_out, anchor(Rh, H_out), anchor(Rw, W_out))


# ------------------------------------------------------------------------------------------------ the batch
def batch(images, first, N, mode, H_out, W_out, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3), resize_size=0, shuffle=1, flip=0, seed=0,
          epoch=0, mean=None, std=None, C_out=None, labels=None):
    """The batch of pcnn_augment_resized_u8_bf16 on images [n][H][W][C] uint8: (x bits [N][H_out][W_out][C_out], labels_out or
    None, i, box (top, left, h, w) int64 [N][4] or None in mode EVAL, flips)"""
    n, H, W, C = images.shape
    C_out = C if C_out is None else C_out
    i = A.indices(n, first, N, shuffle, seed, epoch)
    fl = A.draws(i.astype(np.uint64), 0, flip, seed, epoch)[2] if flip else np.zeros(N, bool)
    u = np.zeros((N, H_out, W_out, C), np.uint8)
    box = None
    if mode == TRAIN:
        box = np.stack(boxes(i.astype(np.uint64), H, W, scale, ratio, seed, epoch)[:4], -1)
        for j in range(N):
            t, l, h, w = box[j]
            u[j] = resample(images[i[j], t:t + h, l:l + w], H_out, W_out)
    else:
        for j in range(N):
            u[j] = eval_image(images[i[j]], resize_size, H_out, W_out)
    u = np.where(fl[:, None, None, None], u[:, :, ::-1], u)
    lut = A.table(C, mean, std)
    x = np.zeros((N, H_out, W_out, C_out), np.uint16)
    for c in range(C):
        x[..., c] = lut[c][u[..., c]]
    return x, (None if labels is None else np.asarray(labels)[i]), i, box, fl
