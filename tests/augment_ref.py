"""numpy replay of the input pipeline (pcnn_augment_u8_bf16, include/pcnn.h): the Feistel permutation of an epoch with its cycle
walk, the crop and flip draws of each image, the ToTensor + Normalize table, and the batch x [N][H][W][C_out] as bf16 bits.

Philox4x32-10 is dropout_ref's; the counters carry the domain bits of pcnn.h in word 1."""
import numpy as np
import torch

from dropout_ref import LO, S32, philox4x32_10
from se_ref import bf16

DOMAIN_AUG, DOMAIN_PERM = 0x80000000, 0x40000000
ROUNDS = 6                  # 4 rounds leave the first position up to 8 sigma off uniform at n = 6 over 50000 epochs


def half_width(n):
    """b: the least with 4^b >= n (2b bits hold every index)"""
    b = 0
    while 4 ** b < n:
        b += 1
    return b


def _key(seed):
    return (seed & 0xFFFFFFFF, seed >> 32)


def _words(a):
    a = np.asarray(a, np.uint64)
    return a & LO, a >> S32


def round_counters(R, r, epoch):
    """the counter words of round r's function at the half values R (uint64 array; epoch an int or an array of R's shape)"""
    return (np.asarray(R, np.uint64), DOMAIN_AUG | DOMAIN_PERM | r, *_words(epoch))


def crop_counters(i, epoch):
    """the counter words of image i's crop and flip draws (i a uint64 array)"""
    lo, hi = _words(i)
    return (lo, hi | np.uint64(DOMAIN_AUG), *_words(epoch))


def feistel(v, seed, epoch, b):
    """one application of the ROUNDS-round network to v (uint64 array of 2b-bit values)"""
    mask = np.uint64((1 << b) - 1)
    L, R = v >> np.uint64(b), v & mask
    for r in range(ROUNDS):
        f = philox4x32_10(round_counters(R, r, epoch), _key(seed))[..., 0].astype(np.uint64) & mask
        L, R = R, L ^ f
    return (L << np.uint64(b)) | R


def permute(e, n, seed, epoch, walks=False):
    """pi(e) for epoch positions e (ints or an array) of a dataset of n images, in one epoch or in an array of epochs of e's
    shape; with walks, also the applications each took"""
    e = np.asarray(e, np.uint64)
    epoch = np.broadcast_to(np.asarray(epoch, np.uint64), e.shape)
    b = half_width(n)
    v = feistel(e.copy(), seed, epoch, b)
    count = np.ones(e.shape, np.int64)
    todo = np.nonzero(v >= np.uint64(n))
    while todo[0].size:
        w = feistel(v[todo], seed, epoch[todo], b)
        v[todo] = w
        count[todo] += 1
        keep = w >= np.uint64(n)
        todo = tuple(t[keep] for t in todo)
    return (v, count) if walks else v


def draws(i, pad, flip, seed, epoch):
    """(oy, ox, flip) of images i: umulhi(w.x, 2 pad + 1), umulhi(w.y, 2 pad + 1), flip and w.z >> 31"""
    w = philox4x32_10(crop_counters(i, epoch), _key(seed)).astype(np.uint64)
    span = np.uint64(2 * pad + 1)
    oy = ((w[..., 0] * span) >> S32).astype(np.int64)
    ox = ((w[..., 1] * span) >> S32).astype(np.int64)
    fl = (w[..., 2] >> np.uint64(31)).astype(bool) & bool(flip)
    return oy, ox, fl


def table(C, mean=None, std=None):
    """uint16 [C][256]: bf16 bits of RN(RN(RN(u / 255) - mean[c]) / std[c]) (mean None = 0, std None = 1)"""
    m = np.zeros(C, np.float32) if mean is None else np.broadcast_to(np.asarray(mean, np.float32).reshape(-1), (C,))
    s = np.ones(C, np.float32) if std is None else np.broadcast_to(np.asarray(std, np.float32).reshape(-1), (C,))
    u = np.arange(256, dtype=np.float32)[None, :]
    with np.errstate(all="ignore"):
        v = (u / np.float32(255) - m[:, None]) / s[:, None]
    return (bf16(v.astype(np.float32)).view(np.uint32) >> 16).astype(np.uint16)


def indices(n, first, N, shuffle, seed, epoch):
    e = np.arange(first, first + N, dtype=np.uint64)
    return (permute(e, n, seed, epoch) if shuffle else e).astype(np.int64)


def batch(images, first, N, shuffle=1, pad=0, flip=0, seed=0, epoch=0, mean=None, std=None, C_out=None, labels=None):
    """The batch of pcnn_augment_u8_bf16 on images [n][H][W][C] uint8: (x bits [N][H][W][C_out], labels_out or None, i, oy, ox, fl)"""
    n, H, W, C = images.shape
    C_out = C if C_out is None else C_out
    i = indices(n, first, N, shuffle, seed, epoch)
    if pad or flip:
        oy, ox, fl = draws(i.astype(np.uint64), pad, flip, seed, epoch)
    else:
        oy = ox = np.zeros(N, np.int64)
        fl = np.zeros(N, bool)
    src = np.pad(images[i], ((0, 0), (pad, pad), (pad, pad), (0, 0)))         # RandomCrop's zero fill
    rows = oy[:, None] + np.arange(H)[None, :]
    w = np.arange(W)[None, :]
    cols = ox[:, None] + np.where(fl[:, None], W - 1 - w, w)                  # the flip after the crop
    u = src[np.arange(N)[:, None, None], rows[:, :, None], cols[:, None, :]]    # [N][H][W][C]
    lut = table(C, mean, std)
    x = np.zeros((N, H, W, C_out), np.uint16)
    for c in range(C):
        x[..., c] = lut[c][u[..., c]]
    return x, (None if labels is None else np.asarray(labels)[i]), i, oy, ox, fl


def torch_batch(images, i, oy, ox, fl, pad, mean, std, C_out):
    """torch eager on the GPU: the batch of images [n][H][W][C] uint8 (device) at indices i with crop offsets (oy, ox) and flips fl
    as NHWC bf16 [N][H][W][C_out].  The divisors are device tensors, so each division is IEEE (a CPU scalar divisor becomes a
    multiply by its reciprocal)."""
    n, H, W, C = images.shape
    N = len(i)
    t = lambda a, dt=torch.long: (a if torch.is_tensor(a) else torch.as_tensor(np.asarray(a))).to(device=images.device, dtype=dt)
    crop = torch.nn.functional.pad(images[t(i)].permute(0, 3, 1, 2), (pad, pad, pad, pad))    # [N][C][H + 2 pad][W + 2 pad]
    w = torch.arange(W, device=images.device)
    rows = t(oy)[:, None] + torch.arange(H, device=images.device)[None, :]
    cols = t(ox)[:, None] + torch.where(t(fl, torch.bool)[:, None], W - 1 - w[None, :], w[None, :])
    u = crop[torch.arange(N, device=images.device)[:, None, None], :, rows[:, :, None], cols[:, None, :]]     # [N][H][W][C]
    m = t(np.zeros(C) if mean is None else mean, torch.float32)
    s = t(np.ones(C) if std is None else std, torch.float32)
    v = u.float().div(torch.full((C,), 255.0, device=images.device)).sub(m).div(s).to(torch.bfloat16)
    out = torch.zeros((N, H, W, C_out), dtype=torch.bfloat16, device=images.device)
    out[..., :C] = v
    return out
