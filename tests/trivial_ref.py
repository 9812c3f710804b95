"""numpy replay of TrivialAugmentWide / RandomErasing batches (pcnn_augment_trivial_u8_bf16, include/pcnn.h): the per-image draws of
op, bin, sign and erase box, the host table from torchvision's own formulas, every op on the uint8 crop in the order pcnn.h states
(both interpolations), and the batch x [N][h][w][C_out] as bf16 bits.

The geometry, the permutation and the table are augment_ref's and resize_ref's; E is bnact_ref's exp_f32.  numpy float32 and
float64 operations are each one IEEE round to nearest, as the kernel's explicitly rounded ones."""
import math

import numpy as np

import augment_ref as A
import resize_ref as R
from bnact_ref import exp_f32
from dropout_ref import philox4x32_10

OPS = ("Identity", "ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate", "Brightness", "Color", "Contrast", "Sharpness",
       "Posterize", "Solarize", "AutoContrast", "Equalize")
SIGNED = {"ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate", "Brightness", "Color", "Contrast", "Sharpness"}
BINS = 31
NONE, NEAREST, BILINEAR = 0, 1, 2
TA_DOMAIN = 0xC0000000
f32 = np.float32


# ------------------------------------------------------------------------------------------------ draws
def counters(i, k, epoch):
    """the counter words of trivial block k of images i (uint64 array)"""
    lo, hi = A._words(i)
    return (lo, hi | np.uint64(TA_DOMAIN | (16 + k) << 24), *A._words(epoch))


def unit24(u):
    return (np.asarray(u, np.uint64) >> np.uint64(8)).astype(f32) * f32(2.0 ** -24)


def draws(i, seed, epoch):
    """(op, bin, sign, u_erase) of images i: umulhi(x, 14), umulhi(y, 31), z >> 31 and U(w) of block 0"""
    i = np.asarray(i, np.uint64)
    b = philox4x32_10(counters(i, 0, epoch), A._key(seed))
    return R.umulhi(b[..., 0], 14), R.umulhi(b[..., 1], BINS), (b[..., 2] >> np.uint32(31)).astype(np.int64), unit24(b[..., 3])


def erase_draws(i, scale, ratio, seed, epoch):
    """(s, lr, w_top, w_left) of images i: the 10 attempts' fp32 draws [len(i)][10] and the randint words of block 6"""
    i = np.asarray(i, np.uint64)
    s0, sr, l0, lrg = R.box_constants(scale, ratio)
    blocks = [philox4x32_10(counters(i, 1 + k, epoch), A._key(seed)) for k in range(R.ATTEMPTS // 2 + 1)]
    us = np.stack([blocks[t // 2][..., 2 if t & 1 else 0] for t in range(R.ATTEMPTS)], -1)
    ul = np.stack([blocks[t // 2][..., 3 if t & 1 else 1] for t in range(R.ATTEMPTS)], -1)
    last = blocks[R.ATTEMPTS // 2]
    return R.uniform(us, s0, sr), R.uniform(ul, l0, lrg), last[..., 0], last[..., 1]


def choose_erase(h, w, s, lr, w_top, w_left, exp=exp_f32):
    """RandomErasing.get_params on the draws: (top, left, eh, ew, attempt), attempt -1 (no erase) when none fits"""
    s, lr = np.asarray(s, f32), np.asarray(lr, f32)
    shape = s.shape[:-1]
    area = float(h * w)
    eh, ew = np.zeros(shape, np.int64), np.zeros(shape, np.int64)
    attempt = np.full(shape, -1, np.int64)
    for t in range(R.ATTEMPTS):
        aspect = np.asarray(exp(lr[..., t]), f32).astype(np.float64)
        ea = area * s[..., t].astype(np.float64)
        with np.errstate(all="ignore"):
            ch, cw = np.rint(np.sqrt(ea * aspect)), np.rint(np.sqrt(ea / aspect))
        ok = (attempt < 0) & (ch < h) & (cw < w)
        eh = np.where(ok, np.nan_to_num(ch).astype(np.int64), eh)
        ew = np.where(ok, np.nan_to_num(cw).astype(np.int64), ew)
        attempt = np.where(ok, t, attempt)
    top = np.where(attempt >= 0, R.umulhi(w_top, np.maximum(h - eh + 1, 1)), 0)
    left = np.where(attempt >= 0, R.umulhi(w_left, np.maximum(w - ew + 1, 1)), 0)
    return top, left, eh, ew, attempt


# ------------------------------------------------------------------------------------------------ the host table
def magnitudes():
    """{op: (fp32 magnitudes [31] or None, signed)} from torchvision's own _augmentation_space"""
    from torchvision.transforms import autoaugment as aa
    space = aa.TrivialAugmentWide()._augmentation_space(BINS)
    return {k: (v.numpy().astype(np.float64) if v.ndim else None, s) for k, (v, s) in space.items()}


def magnitude(mags, op, b, sign):
    m, signed = mags[OPS[op]]
    v = 0.0 if m is None else float(m[b])
    return -v if signed and sign else v


def entry(mags, op, b, sign, h, w):
    """the table entry float32 [6] of (op, bin, sign) for an h x w crop, by torchvision's formulas"""
    import torchvision.transforms.functional as F
    name, mag = OPS[op], magnitude(mags, op, b, sign)
    e = np.zeros(6, f32)
    if name in ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate"):
        if name in ("ShearX", "ShearY"):
            shear = [math.degrees(math.atan(mag)), 0.0] if name == "ShearX" else [0.0, math.degrees(math.atan(mag))]
            m = F._get_inverse_affine_matrix([1.0 * (0 - w * 0.5), 1.0 * (0 - h * 0.5)], 0.0, [0.0, 0.0], 1.0, shear)
        elif name == "Rotate":
            m = F._get_inverse_affine_matrix([0.0, 0.0], -mag, [0.0, 0.0], 1.0, [0.0, 0.0])
        else:
            t = [1.0 * int(mag), 0.0] if name == "TranslateX" else [0.0, 1.0 * int(mag)]
            m = F._get_inverse_affine_matrix([0.0, 0.0], 0.0, t, 1.0, [0.0, 0.0])
        th = np.asarray(m, f32)
        e[:3] = th[:3] / f32(0.5 * w)
        e[3:] = th[3:] / f32(0.5 * h)
    elif name in ("Brightness", "Color", "Contrast", "Sharpness"):
        ratio = 1.0 + mag
        e[0], e[1] = f32(ratio), f32(1.0 - ratio)
    elif name == "Posterize":
        e[0] = (-int(2 ** (8 - int(mag)))) & 255
    elif name == "Solarize":
        e[0] = math.ceil(f32(mag))
    return e


def table(h, w):
    """float32 [14][31][2][6]"""
    mags = magnitudes()
    return np.array([[[entry(mags, op, b, s, h, w) for s in range(2)] for b in range(BINS)] for op in range(len(OPS))], f32)


# ------------------------------------------------------------------------------------------------ the ops on uint8 [h][w][C]
def blend(a, b, e):
    v = f32(e[0]) * np.asarray(a, f32) + f32(e[1]) * np.asarray(b, f32)
    return np.clip(v, 0, 255).astype(np.uint8)


def gray(img):
    img = img.astype(f32)
    return ((f32(0.2989) * img[..., 0] + f32(0.587) * img[..., 1]) + f32(0.114) * img[..., 2]).astype(np.uint8)


def grid_coords(h, w, e):
    """(ix, iy) float32 [h][w]: the grid of the rescaled matrix unnormalised to pixels, in pcnn.h's order"""
    bx = (np.arange(w, dtype=f32) + f32(0.5 - 0.5 * w))[None, :]
    by = (np.arange(h, dtype=f32) + f32(0.5 - 0.5 * h))[:, None]
    gx = (bx * f32(e[0]) + by * f32(e[1])) + f32(e[2])
    gy = (bx * f32(e[3]) + by * f32(e[4])) + f32(e[5])
    ix = (gx + f32(1)) * f32(0.5 * w) - f32(0.5)
    iy = (gy + f32(1)) * f32(0.5 * h) - f32(0.5)
    return ix.astype(f32), iy.astype(f32)


def sample(img, ix, iy, interp):
    h, w, C = img.shape

    def at(fy, fx):
        ok = (fx >= 0) & (fx < w) & (fy >= 0) & (fy < h)
        yy, xx = np.where(ok, fy, 0).astype(np.int64), np.where(ok, fx, 0).astype(np.int64)
        return np.where(ok[..., None], img[yy, xx].astype(f32), f32(0))

    if interp == NEAREST:
        return at(np.rint(iy), np.rint(ix)).astype(np.uint8)
    x0, y0 = np.floor(ix), np.floor(iy)
    tw = ix - x0
    te = f32(1) - tw
    tn = iy - y0
    ts = f32(1) - tn
    wt = lambda a, b: (a * b)[..., None]
    v = at(y0, x0) * wt(ts, te)
    v = v + at(y0, x0 + f32(1)) * wt(ts, tw)
    v = v + at(y0 + f32(1), x0) * wt(tn, te)
    v = v + at(y0 + f32(1), x0 + f32(1)) * wt(tn, tw)
    return np.minimum(np.rint(v), 255).astype(np.uint8)


def blurred(img):
    """_blurred_degenerate_image in pcnn.h's order: interior rint(RN sum of RN(k u), row-major taps), border unchanged"""
    h, w, C = img.shape
    out = img.copy()
    if h <= 2 or w <= 2:
        return out
    x = img.astype(f32)
    w1, w5 = f32(1) / f32(13), f32(5) / f32(13)
    acc = None
    for k in range(9):
        dy, dx = k // 3, k % 3
        t = (w5 if k == 4 else w1) * x[dy:h - 2 + dy, dx:w - 2 + dx]
        acc = t if acc is None else (acc + t).astype(f32)
    out[1:-1, 1:-1] = np.minimum(np.rint(acc), 255).astype(np.uint8)
    return out


def equalize_channel(ch):
    hist = np.bincount(ch.reshape(-1), minlength=256).astype(np.int64)
    nz = hist[hist != 0]
    step = int(nz[:-1].sum()) // 255
    if step == 0:
        return ch
    lut = (np.cumsum(hist) + step // 2) // step
    lut = np.clip(np.concatenate([[0], lut[:-1]]), 0, 255)
    return lut[ch].astype(np.uint8)


def apply_op(img, op, e, interp):
    """op (an index into OPS) with table entry e on one uint8 crop [h][w][C], C 1 or 3"""
    name = OPS[op]
    h, w, C = img.shape
    if name in ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate"):
        ix, iy = grid_coords(h, w, e)
        return sample(img, ix, iy, interp)
    if name == "Brightness":
        return blend(img, 0, e)
    if name == "Color":
        return blend(img, gray(img)[..., None], e) if C == 3 else img
    if name == "Contrast":
        g = gray(img) if C == 3 else img[..., 0]
        mean = f32(np.int64(g.astype(np.int64).sum())) / f32(h * w)
        return blend(img, mean, e)
    if name == "Sharpness":
        return img if h <= 2 or w <= 2 else blend(img, blurred(img), e)
    if name == "Posterize":
        return img & np.uint8(int(e[0]))
    if name == "Solarize":
        return np.where(img >= int(e[0]), 255 - img, img).astype(np.uint8)
    if name == "AutoContrast":
        lo = img.min(axis=(0, 1)).astype(f32)
        hi = img.max(axis=(0, 1)).astype(f32)
        flat = hi == lo
        with np.errstate(divide="ignore"):
            scale = np.where(flat, f32(1), (f32(1) / np.where(flat, f32(1), hi - lo)) * f32(255)).astype(f32)
        lo = np.where(flat, f32(0), lo)
        return np.clip((img.astype(f32) - lo) * scale, 0, 255).astype(np.uint8)
    if name == "Equalize":
        return np.stack([equalize_channel(img[..., c]) for c in range(C)], -1)
    return img


# ------------------------------------------------------------------------------------------------ the batch
def crops(images, first, N, shuffle=1, pad=0, flip=0, seed=0, epoch=0, crop_size=None, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3)):
    """(u [N][h][w][C] uint8, i): the geometry's bytes, augment_ref's crop or resize_ref's RandomResizedCrop, with the flip"""
    n, H, W, C = images.shape
    i = A.indices(n, first, N, shuffle, seed, epoch)
    if crop_size is None:
        x, _, i, *_ = A.batch(images, first, N, shuffle, pad, flip, seed, epoch)
    else:
        x, _, i, _, _ = R.batch(images, first, N, R.TRAIN, *crop_size, scale, ratio, shuffle=shuffle, flip=flip, seed=seed, epoch=epoch)
    return bytes_of(x), i


def bytes_of(x_bits):
    """the bytes u of x bits formed by the mean 0 / std 1 table (bf16(u / 255) is injective over bytes)"""
    inv = np.zeros(1 << 16, np.uint8)
    inv[A.table(1)[0]] = np.arange(256, dtype=np.uint8)
    return inv[x_bits]


def batch(images, first, N, trivial=NEAREST, erase_p=0.0, erase_scale=(0.02, 0.33), erase_ratio=(0.3, 3.3), crop_size=None,
          scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3), shuffle=1, pad=0, flip=0, seed=0, epoch=0, mean=None, std=None, C_out=None,
          labels=None, tab=None):
    """The batch of pcnn_augment_trivial_u8_bf16: (x bits [N][h][w][C_out], labels_out or None, i, draws dict).  tab is table(h, w)
    when None."""
    n, H, W, C = images.shape
    C_out = C if C_out is None else C_out
    u, i = crops(images, first, N, shuffle, pad, flip, seed, epoch, crop_size, scale, ratio)
    h, w = u.shape[1:3]
    tab = table(h, w) if tab is None else tab
    op, b, sign, ue = draws(i.astype(np.uint64), seed, epoch)
    if not trivial:
        op = np.zeros(N, np.int64)
    t = [apply_op(u[j], int(op[j]), tab[op[j], b[j], sign[j]], trivial) for j in range(N)]
    lut = A.table(C, mean, std)
    x = np.zeros((N, h, w, C_out), np.uint16)
    for c in range(C):
        x[..., c] = lut[c][np.stack(t)[..., c]] if N else 0
    erase = (ue < f32(erase_p)) if erase_p > 0 else np.zeros(N, bool)
    box = np.zeros((N, 4), np.int64)
    if erase_p > 0:
        top, left, eh, ew, attempt = choose_erase(h, w, *erase_draws(i.astype(np.uint64), erase_scale, erase_ratio, seed, epoch))
        erase &= attempt >= 0
        box = np.stack([top, left, eh, ew], -1)
        for j in np.nonzero(erase)[0]:
            tp, lf, eh_, ew_ = box[j]
            x[j, tp:tp + eh_, lf:lf + ew_, :C] = 0
    return x, (None if labels is None else np.asarray(labels)[i]), i, dict(op=op, bin=b, sign=sign, erase=erase, box=box)
