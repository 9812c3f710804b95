"""numpy replay of mixed batches and soft targets (pcnn_augment_mix_u8_bf16, pcnn_softmax_ce_soft_bf16, ImageBatcher's
mixup_alpha / cutmix_alpha; include/pcnn.h): the host draws of a batch, the MixUp or CutMix batch built on augment_ref's
permutation, draws and table plus the fp32 table, and the soft-target softmax cross-entropy (float64 g, loss and pred, and the
fp32 target q), and torch's eager fp32 batch that torchvision's MixUp and CutMix take."""
import math

import numpy as np
import torch

import augment_ref as A
from se_ref import bf16

MIXUP, CUTMIX = 1, 2


def cutmix_box(lam, r_x, r_y, H, W):
    """(box (x1, y1, x2, y2), lam_adjusted) as torchvision's v2.CutMix.make_params forms them from lam and the centre"""
    r = 0.5 * math.sqrt(1.0 - lam)
    r_w_half, r_h_half = int(r * W), int(r * H)
    x1, y1 = max(r_x - r_w_half, 0), max(r_y - r_h_half, 0)
    x2, y2 = min(r_x + r_w_half, W), min(r_y + r_h_half, H)
    return (x1, y1, x2, y2), float(1.0 - (x2 - x1) * (y2 - y1) / (W * H))


def draws(seed, epoch, step, H, W, mixup_alpha, cutmix_alpha):
    """(kind, lam, box, weight, centre) of training batch `step` of `epoch`: numpy's Philox keyed by seed at counter (0, 0, epoch,
    step); CutMix iff random() < 1/2 when both alphas are > 0; lam = beta(alpha, alpha); for CutMix r_x = integers(W), then
    r_y = integers(H).  weight is the weight of labels: lam for MixUp, lam_adjusted for CutMix.  box and centre None for MixUp."""
    rng = np.random.Generator(np.random.Philox(key=int(seed), counter=np.array([0, 0, int(epoch), int(step)], np.uint64)))
    if mixup_alpha > 0 and cutmix_alpha > 0:
        cutmix = rng.random() < 0.5
    else:
        cutmix = cutmix_alpha > 0
    alpha = cutmix_alpha if cutmix else mixup_alpha
    lam = float(rng.beta(alpha, alpha))
    if not cutmix:
        return "mixup", lam, None, lam, None
    r_x = int(rng.integers(W))
    r_y = int(rng.integers(H))
    box, lam_adjusted = cutmix_box(lam, r_x, r_y, H, W)
    return "cutmix", lam, box, lam_adjusted, (r_x, r_y)


def ftable(C, mean=None, std=None):
    """float32 [C][256]: RN(RN(RN(u / 255) - mean[c]) / std[c]), the values augment_ref.table rounds to bf16"""
    m = np.zeros(C, np.float32) if mean is None else np.broadcast_to(np.asarray(mean, np.float32).reshape(-1), (C,))
    s = np.ones(C, np.float32) if std is None else np.broadcast_to(np.asarray(std, np.float32).reshape(-1), (C,))
    u = np.arange(256, dtype=np.float32)[None, :]
    with np.errstate(all="ignore"):
        return ((u / np.float32(255) - m[:, None]) / s[:, None]).astype(np.float32)


def source_bytes(images, i, oy, ox, fl, pad):
    """uint8 [N][H][W][C]: the cropped and flipped source bytes of images i (augment_ref.batch's geometry)"""
    n, H, W, C = images.shape
    N = len(i)
    src = np.pad(images[i], ((0, 0), (pad, pad), (pad, pad), (0, 0)))
    rows = oy[:, None] + np.arange(H)[None, :]
    w = np.arange(W)[None, :]
    cols = ox[:, None] + np.where(fl[:, None], W - 1 - w, w)
    return src[np.arange(N)[:, None, None], rows[:, :, None], cols[:, None, :]]


def partner(N):
    """j' = (j + N - 1) mod N for every batch position j (torchvision's roll(1, 0))"""
    return (np.arange(N) + N - 1) % N


def bits_of(f32):
    return (bf16(np.asarray(f32, np.float32)).view(np.uint32) >> 16).astype(np.uint16)


def batch(images, first, N, mode, lam, box=(0, 0, 0, 0), shuffle=1, pad=0, flip=0, seed=0, epoch=0, mean=None, std=None, C_out=None,
          labels=None):
    """The batch of pcnn_augment_mix_u8_bf16 on images [n][H][W][C] uint8: (x bits [N][H][W][C_out], labels_out, labels_b_out)
    (the labels None without labels)"""
    n, H, W, C = images.shape
    C_out = C if C_out is None else C_out
    plain, lab, i, oy, ox, fl = A.batch(images, first, N, shuffle, pad, flip, seed, epoch, mean, std, C_out, labels)
    jb = partner(N)
    if mode == MIXUP:
        u = source_bytes(images, i, oy, ox, fl, pad)
        ft = ftable(C, mean, std)
        a = np.stack([ft[c][u[..., c]] for c in range(C)], axis=-1)
        b = a[jb]
        mixed = b * np.float32(1.0 - lam) + a * np.float32(lam)          # float32: each product and the sum rounded, no FMA
        x = np.zeros((N, H, W, C_out), np.uint16)
        x[..., :C] = bits_of(mixed)
    else:
        x1, y1, x2, y2 = box
        x = plain.copy()
        x[:, y1:y2, x1:x2] = plain[jb][:, y1:y2, x1:x2]
    return x, lab, (None if lab is None else lab[jb])


def soft_target(labels, labels_b, lam, eps, O):
    """(m, q) float32 [N][O]: m = RN(RN(onehot(labels_b) RN32(1 - lam)) + RN(onehot(labels) RN32(lam))) (labels_b None:
    onehot(labels)), q = RN(RN(m RN32(1 - eps)) + RN32(eps / O)).  Labels >= O have no one."""
    labels = np.asarray(labels).astype(np.int64)
    N = len(labels)
    onehot = lambda y: (np.arange(O)[None, :] == np.asarray(y).astype(np.int64)[:, None]).astype(np.float32)
    m = onehot(labels)
    if labels_b is not None:
        m = onehot(labels_b) * np.float32(1.0 - lam) + m * np.float32(lam)
    q = m * np.float32(1.0 - eps) + np.float32(eps / O)
    assert m.shape == (N, O)
    return m.astype(np.float32), q.astype(np.float32)


def softmax_ce_soft_f64(z, labels, labels_b, lam, eps, scale):
    """(g, loss, pred, q): g = (softmax(z) - q) * scale, loss = -sum_t q_t ((z_t - m) - log den) over the terms with q_t != 0, in
    float64; pred the first argmax.  A row holding NaN: g and loss NaN, pred -1.  A label or label_b >= O: g and loss NaN."""
    z = np.asarray(z, np.float64)
    N, O = z.shape
    labels = np.asarray(labels).astype(np.int64)
    _, q = soft_target(labels, labels_b, lam, eps, O)
    q64 = q.astype(np.float64)
    m = z.max(axis=1, keepdims=True)
    with np.errstate(invalid="ignore", over="ignore"):
        e = np.exp(z - m)
        den = e.sum(axis=1, keepdims=True)
        g = (e / den - q64) * scale
        terms = np.where(q64 != 0, q64 * ((z - m) - np.log(den)), 0.0)
    loss = -terms.sum(axis=1)
    nan = np.isnan(z).any(axis=1)
    bad = nan | (labels >= O)
    if labels_b is not None:
        bad |= np.asarray(labels_b).astype(np.int64) >= O
    g[bad] = np.nan
    loss[bad] = np.nan
    pred = np.where(nan, -1, np.argmax(np.where(np.isnan(z), -np.inf, z), axis=1))
    return g, loss, pred, q


def torch_f32_batch(images, i, oy, ox, fl, pad, mean, std):
    """torch eager on the GPU: the fp32 NCHW batch ToTensor + Normalize give before any bf16 rounding (augment_ref.torch_batch's
    operations)"""
    n, H, W, C = images.shape
    t = lambda a, dt=torch.long: torch.as_tensor(np.asarray(a)).to(device=images.device, dtype=dt)
    crop = torch.nn.functional.pad(images[t(i)].permute(0, 3, 1, 2), (pad, pad, pad, pad))
    w = torch.arange(W, device=images.device)
    rows = t(oy)[:, None] + torch.arange(H, device=images.device)[None, :]
    cols = t(ox)[:, None] + torch.where(t(fl, torch.bool)[:, None], W - 1 - w[None, :], w[None, :])
    u = crop[torch.arange(len(i), device=images.device)[:, None, None], :, rows[:, :, None], cols[:, None, :]]     # [N][H][W][C]
    m = t(np.zeros(C) if mean is None else mean, torch.float32)
    s = t(np.ones(C) if std is None else std, torch.float32)
    return u.float().div(torch.full((C,), 255.0, device=images.device)).sub(m).div(s).permute(0, 3, 1, 2).contiguous()
