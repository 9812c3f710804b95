"""References of the image-to-image regression operations (TEST INFRASTRUCTURE ONLY): pixel shuffle and unshuffle
(pcnn_pixel_shuffle_nhwc_bf16 / pcnn_pixel_unshuffle_nhwc_bf16) as numpy permutations of bf16 bits, and the regression losses
(pcnn_regression_loss_bf16) replayed in float32 at include/pcnn.h's rounding points, so the device must give their bits.
test_restore_cpu.py pins them to torch's pixel_shuffle, pixel_unshuffle, mse_loss and l1_loss.

Layouts are NHWC: the coarse map [N][H][W][C r^2], the fine map [N][H r][W r][C]."""
import numpy as np

F32 = np.float32
MSE, L1 = 0, 1


def shuffle(x, r):
    """fine[n][h r + i][w r + j][c] = x[n][h][w][c r^2 + i r + j] for any array x [N][H][W][C r^2] (bits or values)"""
    N, H, W, Crr = x.shape
    C = Crr // (r * r)
    return x.reshape(N, H, W, C, r, r).transpose(0, 1, 4, 2, 5, 3).reshape(N, H * r, W * r, C)


def unshuffle(x, r):
    """the inverse of shuffle: x [N][H][W][C] -> [N][H / r][W / r][C r^2]"""
    N, H, W, C = x.shape
    return x.reshape(N, H // r, r, W // r, r, C).transpose(0, 1, 3, 5, 2, 4).reshape(N, H // r, W // r, C * r * r)


def depth_to_space(x, r):
    """TensorFlow's channel order, fine[n][h r + i][w r + j][c] = x[n][h][w][(i r + j) C + c]: not the op's permutation"""
    N, H, W, Crr = x.shape
    C = Crr // (r * r)
    return x.reshape(N, H, W, r, r, C).transpose(0, 1, 3, 2, 4, 5).reshape(N, H * r, W * r, C)


def bf16_bits(f32):
    """the device's bf16_rn: round to nearest even, every NaN written as 0x7FFF"""
    u = np.ascontiguousarray(f32, F32).view(np.uint32).astype(np.uint64)
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    return np.where(nan, 0x7FFF, (u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def bits_f32(bits):
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(F32)


def loss_replay(pred_bits, target_bits, C, mode, scale, target_stride=None):
    """(dpred bits [pixels][C], loss float32 [pixels]) of the device call on bf16 bits pred [pixels][C] and target
    [pixels][target_stride] (None = C): d = RN32(p - t); MSE: term RN32(d d), dpred bf16_rn(RN32(RN32(2 scale) d)); L1: term |d|,
    dpred bf16_rn(RN32(s(d) scale)) with s = +1, -1 or +0 (d = +-0, NaN); loss the fp32 sum from +0 of the terms in ascending c."""
    ts = C if target_stride is None else target_stride
    p = bits_f32(pred_bits).reshape(-1, C)
    t = bits_f32(target_bits).reshape(-1, ts)[:, :C]
    scale = F32(scale)
    with np.errstate(all="ignore"):
        d = p - t
        if mode == MSE:
            term, g = d * d, (F32(2) * scale) * d
        else:
            s = np.where(d > 0, F32(1), np.where(d < 0, F32(-1), F32(0))).astype(F32)
            term, g = np.abs(d), s * scale
        loss = np.zeros(p.shape[0], F32)
        for c in range(C):
            loss = loss + term[:, c]
    return bf16_bits(g), loss
