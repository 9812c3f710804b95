"""References of the dense-prediction operations (TEST INFRASTRUCTURE ONLY): the transposed convolution (pcnn_conv_transpose_fwd and
its gradients), the bilinear resize (pcnn_upsample_bilinear_nhwc_bf16_fwd / _bwd), the per-pixel cross-entropy
(pcnn_softmax_ce_pixels_bf16) and the mask batch (pcnn_augment_mask_u8).  float64 references are pinned to torch by
test_segment_cpu.py; the float32 replays follow include/pcnn.h's order of operations, so the device must give their bits.

Layouts are NHWC; torch's ConvTranspose2d weight is [C_in][C_out][R][S]."""
import numpy as np

import augment_ref
import linear_ref

F32 = np.float32


# ------------------------------------------------------------------------------------------------ transposed convolution
def convt_out(H, W, R, S, stride, padding=(0, 0), output_padding=(0, 0)):
    return ((H - 1) * stride - 2 * padding[0] + R + output_padding[0], (W - 1) * stride - 2 * padding[1] + S + output_padding[1])


def convt_fwd_f64(x, w, b=None, stride=1, padding=(0, 0), output_padding=(0, 0), act=0):
    """(pre, y) of conv_transpose2d in float64: x [N][H][W][C_in], w [C_in][C_out][R][S]; act 0 none, 1 sigmoid, 3 ReLU"""
    x, w = np.asarray(x, np.float64), np.asarray(w, np.float64)
    N, H, W, _ = x.shape
    _, Co, R, S = w.shape
    Ho, Wo = convt_out(H, W, R, S, stride, padding, output_padding)
    canvas = np.zeros((N, (H - 1) * stride + R + output_padding[0], (W - 1) * stride + S + output_padding[1], Co))
    for r in range(R):
        for s in range(S):
            canvas[:, r:r + (H - 1) * stride + 1:stride, s:s + (W - 1) * stride + 1:stride] += np.einsum("nijc,cd->nijd", x, w[:, :, r, s])
    pre = canvas[:, padding[0]:padding[0] + Ho, padding[1]:padding[1] + Wo].copy()
    if b is not None:
        pre = pre + np.asarray(b, np.float64)
    return pre, act_f64(pre, act)


def act_f64(pre, act):
    if act == 1:
        return 1.0 / (1.0 + np.exp(-pre))
    if act == 3:
        return np.where(pre < 0, 0.0, pre)
    return pre


def convt_bwd_f64(x, w, dpre, stride=1, padding=(0, 0)):
    """(dx, dw, db) of conv_transpose2d in float64 from the gradient dpre [N][H_out][W_out][C_out] at the pre-activation"""
    x, w, dpre = (np.asarray(a, np.float64) for a in (x, w, dpre))
    N, H, W, _ = x.shape
    _, Co, R, S = w.shape
    Ho, Wo = dpre.shape[1:3]
    canvas = np.zeros((N, max((H - 1) * stride + R, padding[0] + Ho), max((W - 1) * stride + S, padding[1] + Wo), Co))
    canvas[:, padding[0]:padding[0] + Ho, padding[1]:padding[1] + Wo] = dpre
    dx = np.zeros(x.shape)
    dw = np.zeros(w.shape)
    for r in range(R):
        for s in range(S):
            d = canvas[:, r:r + (H - 1) * stride + 1:stride, s:s + (W - 1) * stride + 1:stride]
            dx += np.einsum("nijd,cd->nijc", d, w[:, :, r, s])
            dw[:, :, r, s] = np.einsum("nijc,nijd->cd", x, d)
    return dx, dw, dpre.sum(axis=(0, 1, 2))


# ------------------------------------------------------------------------------------------------ bilinear resize
def axis_taps(n_in, n_out, dtype=F32):
    """(i0, i1, l0, l1) of every output index, in `dtype` arithmetic by include/pcnn.h's rule (float32: the device's; float64:
    torch's CPU float64 path)"""
    d = np.arange(n_out)
    if n_in == n_out:
        return d.copy(), d.copy(), np.ones(n_out, dtype), np.zeros(n_out, dtype)
    scale = dtype(dtype(n_in) / dtype(n_out))
    real = (scale * (d.astype(dtype) + dtype(0.5))).astype(dtype) - dtype(0.5)
    real = np.where(real < 0, dtype(0), real).astype(dtype)
    i0 = np.minimum(np.floor(real).astype(np.int64), n_in - 1)
    l1 = np.clip((real - i0.astype(dtype)).astype(dtype), dtype(0), dtype(1)).astype(dtype)
    l0 = (dtype(1) - l1).astype(dtype)
    i1 = i0 + (i0 < n_in - 1)
    return i0, i1, l0, l1


def resize_matrix(n_in, n_out):
    """A [n_out][n_in] of the float64 weights: y = A_h x A_w^T per channel"""
    i0, i1, l0, l1 = axis_taps(n_in, n_out, np.float64)
    A = np.zeros((n_out, n_in))
    np.add.at(A, (np.arange(n_out), i0), l0)
    np.add.at(A, (np.arange(n_out), i1), l1)
    return A


def upsample_fwd_f64(x, Ho, Wo):
    x = np.asarray(x, np.float64)
    return np.einsum("hi,nijc,wj->nhwc", resize_matrix(x.shape[1], Ho), x, resize_matrix(x.shape[2], Wo))


def upsample_bwd_f64(dy, H, W):
    dy = np.asarray(dy, np.float64)
    return np.einsum("hi,nhwc,wj->nijc", resize_matrix(H, dy.shape[1]), dy, resize_matrix(W, dy.shape[2]))


def bf16_bits(f32):
    """the device's bf16_rn: round to nearest even, every NaN written as __float2bfloat16_rn writes it, 0x7FFF"""
    import pcnn_loader
    f32 = np.asarray(f32, F32)
    return np.where(np.isnan(f32), np.uint16(0x7FFF), pcnn_loader.load().f32_to_bf16_bits(f32)).astype(np.uint16)


def bits_f32(bits):
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(F32)


def upsample_fwd_replay(x_bits, Ho, Wo):
    """bf16 bits of the device forward on bf16 bits x [N][H][W][C]"""
    x = bits_f32(x_bits)
    N, H, W, C = x.shape
    hi0, hi1, hl0, hl1 = axis_taps(H, Ho)
    wi0, wi1, wl0, wl1 = axis_taps(W, Wo)
    g = lambda ri, ci: x[:, ri][:, :, ci]
    wl0, wl1 = wl0[None, None, :, None], wl1[None, None, :, None]
    with np.errstate(all="ignore"):
        top = (wl0 * g(hi0, wi0)).astype(F32) + (wl1 * g(hi0, wi1)).astype(F32)
        bot = (wl0 * g(hi1, wi0)).astype(F32) + (wl1 * g(hi1, wi1)).astype(F32)
        y = (hl0[None, :, None, None] * top).astype(F32) + (hl1[None, :, None, None] * bot).astype(F32)
    return bf16_bits(y)


def _reach(n_in, n_out):
    """per input index the output indices reaching it, ascending, with tap_weight's weight: (idx [n_in][L], wt [n_in][L], ok)"""
    i0, i1, l0, l1 = axis_taps(n_in, n_out)
    lists = [[] for _ in range(n_in)]
    for d in range(n_out):
        if i0[d] == i1[d]:
            lists[i0[d]].append((d, F32(l0[d] + l1[d])))
        else:
            lists[i0[d]].append((d, l0[d]))
            lists[i1[d]].append((d, l1[d]))
    L = max(1, max(len(v) for v in lists))
    idx, wt, ok = np.zeros((n_in, L), np.int64), np.zeros((n_in, L), F32), np.zeros((n_in, L), bool)
    for i, v in enumerate(lists):
        for k, (d, w) in enumerate(v):
            idx[i, k], wt[i, k], ok[i, k] = d, w, True
    return idx, wt, ok


def upsample_bwd_replay(dy_bits, H, W):
    """bf16 bits of the device's gathered backward on bf16 bits dy [N][H_out][W_out][C]"""
    dy = bits_f32(dy_bits)
    N, Ho, Wo, C = dy.shape
    hidx, hw, hok = _reach(H, Ho)
    widx, ww, wok = _reach(W, Wo)
    s = np.zeros((N, H, W, C), F32)
    with np.errstate(all="ignore"):
        for a in range(hidx.shape[1]):
            for b in range(widx.shape[1]):
                wt = (hw[:, a][:, None] * ww[:, b][None, :]).astype(F32)                        # [H][W]
                term = (wt[None, :, :, None] * dy[:, hidx[:, a]][:, :, widx[:, b]]).astype(F32)
                ok = (hok[:, a][:, None] & wok[:, b][None, :])[None, :, :, None]
                s = np.where(ok, (s + term).astype(F32), s)
    return bf16_bits(s)


# ------------------------------------------------------------------------------------------------ per-pixel cross-entropy
def ce_pixels_f64(z, targets, ignore_index):
    """(g, loss, pred, count, mean loss) of cross_entropy(ignore_index) with mean reduction in float64, include/pcnn.h's form:
    each non-ignored row is softmax_ce_f64's at scale fp32(1 / count); ignored rows g = +0 and loss 0"""
    z = np.asarray(z, np.float64)
    t = np.asarray(targets).astype(np.int64)
    ign = t == ignore_index
    count = int((~ign).sum())
    scale = float(F32(1.0 / count)) if count else float("inf")
    with np.errstate(all="ignore"):
        g, loss, pred = linear_ref.softmax_ce_f64(z, t, scale)
    g[ign] = 0.0
    loss[ign] = 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = loss.sum() / count if count else float("nan")
    return g, loss, pred, count, mean


# ------------------------------------------------------------------------------------------------ masks
def mask_batch(masks, first, N, shuffle=1, pad=0, flip=0, seed=0, epoch=0, fill=255):
    """(masks_out [N][H][W], i, oy, ox, fl): the device's mask batch from the image call's draws"""
    n, H, W = masks.shape
    i = augment_ref.indices(n, first, N, shuffle, seed, epoch)
    if pad or flip:
        oy, ox, fl = augment_ref.draws(i.astype(np.uint64), pad, flip, seed, epoch)
    else:
        oy = ox = np.zeros(N, np.int64)
        fl = np.zeros(N, bool)
    src = np.pad(masks[i], ((0, 0), (pad, pad), (pad, pad)), constant_values=fill)
    rows = oy[:, None] + np.arange(H)[None, :]
    w = np.arange(W)[None, :]
    cols = ox[:, None] + np.where(fl[:, None], W - 1 - w, w)
    return src[np.arange(N)[:, None, None], rows[:, :, None], cols[:, None, :]], i, oy, ox, fl


def torchvision_masks(masks, i, oy, ox, fl, pad, fill=255):
    """torchvision v2 RandomCrop(padding=pad, fill={Mask: fill}) + RandomHorizontalFlip on tv_tensors.Mask, with the given draws"""
    import torch
    from torchvision import tv_tensors
    from torchvision.transforms.v2 import functional as TF
    n, H, W = masks.shape
    out = []
    for k in range(len(i)):
        m = tv_tensors.Mask(torch.from_numpy(np.ascontiguousarray(masks[i[k]]))[None])
        m = TF.pad(m, [pad, pad, pad, pad], fill=fill)
        m = TF.crop(m, int(oy[k]), int(ox[k]), H, W)
        if fl[k]:
            m = TF.horizontal_flip(m)
        out.append(m[0].numpy())
    return np.stack(out)


def digit_masks(u8, labels):
    """The golden digits' segmentation targets: pixel >= 128 -> digit + 1, pixel < 32 -> 0 (background), else 255 (ignored)"""
    u8 = np.asarray(u8).reshape(-1, 28, 28)
    m = np.full(u8.shape, 255, np.uint8)
    m[u8 < 32] = 0
    fg = u8 >= 128
    m[fg] = (np.asarray(labels, np.uint8)[:, None, None] + 1).repeat(28, 1).repeat(28, 2)[fg]
    return m
