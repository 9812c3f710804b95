"""numpy replay of dropout and stochastic depth (pcnn_dropout_bf16, include/pcnn.h): a vectorised Philox4x32-10 in uint64
arithmetic, the host's T / scale rule, the mask at each index and the float32 values of y.

x and r are carried as float32 arrays of bf16 values [N][row_elems]; numpy multiplies and adds float32 arrays with one IEEE
rounding each, as the kernel's __fmul_rn / __fadd_rn, and se_ref.bf16 rounds to nearest even as __float2bfloat16_rn."""
import numpy as np

from se_ref import bf16

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
LO = np.uint64(0xFFFFFFFF)
S32 = np.uint64(32)


def philox4x32_10(ctr, key):
    """ctr: 4 uint32 words (ints or arrays of one shape); key: 2 uint32 words (ints) -> uint32 array [..., 4]"""
    c = [np.asarray(w, np.uint64) & LO for w in ctr]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]                  # < 2^64: exact in uint64
        c = [(p1 >> S32) ^ c[1] ^ np.uint64(k0), p1 & LO, (p0 >> S32) ^ c[3] ^ np.uint64(k1), p0 & LO]
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return np.stack(np.broadcast_arrays(*c), -1).astype(np.uint32)


def draws(i, seed, call):
    """uint32 draws at the indices i (uint64 array): word i & 3 of Philox at counter (i >> 2, call), key seed"""
    i = np.asarray(i, np.uint64)
    q = i >> np.uint64(2)
    w = philox4x32_10((q & LO, q >> S32, call & 0xFFFFFFFF, call >> 32), (seed & 0xFFFFFFFF, seed >> 32))
    return np.take_along_axis(w, (i & np.uint64(3)).astype(np.int64)[..., None], -1)[..., 0]


def threshold(p):
    """(T, scale): an element is dropped iff its draw < T; T the uint32 nearest to p 2^32 (ties to even), scale fp32(1 / (1 - p))"""
    T = min(int(np.rint(float(p) * 2.0 ** 32)), 0xFFFFFFFF)
    return T, np.float32(1.0 / (1.0 - float(p)))


def keep(N, row_elems, p, seed, call, per_sample=False):
    """bool [N][row_elems]: True where the element is kept"""
    T, _ = threshold(p)
    if per_sample:
        return np.repeat((draws(np.arange(N, dtype=np.uint64), seed, call) >= T)[:, None], row_elems, 1)
    n = N * row_elems                       # indices 0 .. n - 1: all four words of counters 0 .. ceil(n / 4) - 1, in order
    q = np.arange(-(-n // 4), dtype=np.uint64)
    w = philox4x32_10((q & LO, q >> S32, call & 0xFFFFFFFF, call >> 32), (seed & 0xFFFFFFFF, seed >> 32)).reshape(-1)[:n]
    return (w >= T).reshape(N, row_elems)


def values(x, kept, scale, r=None):
    """y as float32 bf16 values: bf16(x * m), or bf16(r + RN(x * m)), m = kept ? scale : 0"""
    m = np.where(kept, np.float32(scale), np.float32(0.0))
    with np.errstate(all="ignore"):
        v = np.asarray(x, np.float32) * m
        if r is not None:
            v = np.asarray(r, np.float32) + v
    return bf16(v)


def dropout(x, p, seed, call, per_sample=False, r=None):
    """the whole call on x [N][row_elems] (float32 bf16 values) -> (y, kept)"""
    N, E = x.shape
    kept = keep(N, E, p, seed, call, per_sample)
    return values(x, kept, threshold(p)[1], r), kept
