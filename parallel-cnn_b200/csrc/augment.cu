// parallel-cnn_b200/csrc/augment.cu -- the input pipeline of the device-trained networks (pcnn_augment_u8_bf16): positions
// first .. first + N - 1 of an epoch of a uint8 dataset [n][H][W][C] in device memory become one bf16 batch in the x layout every
// plan reads, [N][image_rows][row_pitch] with H x W pixels of C_out channels, plus the batch's labels.  Position e of the epoch
// is image pi(e), pi a keyed Feistel permutation of [0, n); image i gets torchvision's RandomCrop(padding = pad, fill = 0) and
// RandomHorizontalFlip from one Philox4x32-10 block, then ToTensor + Normalize through a 256-entry table per channel that the
// host forms.  The contract, every operation in its order, is in include/pcnn.h.
//
// pcnn_augment_mix_u8_bf16 is the same pipeline with torchvision's MixUp or CutMix of each image j and its partner
// j' = (j + N - 1) mod N (roll(1, 0)): k_augment's MODE 1 and 2 instantiations, in which lane 0 of warp 1 walks and draws the partner
// beside thread 0's own walk and draw, and each element is formed from both images' bytes.
//
// A CTA takes one (batch position, block of output rows) unit: thread 0 walks the permutation and draws the crop, and the CTA
// writes the rows, as 16-byte vectors of 8 elements when W C_out % 8 == 0 (and the pitch is then a multiple of 8), otherwise as
// single elements, reading the source bytes straight from global memory (no alignment is assumed of an image's base).  The
// grid, a function of the shape alone, loops over the units; no atomics, so every run on every H100 gives the same bits.
#include "pcnn_internal.h"
#include "philox.cuh"

#include <cuda_bf16.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <type_traits>

namespace {

constexpr int AUG_THREADS = 256;
constexpr long long AUG_MAX_GRID = 1 << 20;     // the units loop past it; no shape a user trains on comes near
constexpr int AUG_CTA_BYTES = 16384;           // output bytes of one unit: rows per CTA = ceil(16 KB / output row), 1 .. H
constexpr unsigned DOMAIN_AUG = 0x80000000u;   // counter word 1: set in every augmentation counter, never in a dropout counter
constexpr unsigned DOMAIN_PERM = 0x40000000u;  // counter word 1: set in the permutation's rounds, never in a crop counter
constexpr int FEISTEL_ROUNDS = 6;             // 4 leave pi(0) 8 sigma off uniform at n = 6 (b = 2) over 50000 epochs

struct AugArgs {
    const uint8_t *img;       // [n][H][W][C]
    const uint8_t *lab;       // [n] or NULL
    __nv_bfloat16 *x;         // [N][image_rows][pitch]
    uint8_t *lab_out;         // [N] or NULL
    long long n, first, img_bytes;   // img_bytes = H W C
    long long units;          // N row_blocks
    int H, W, C, C_out, pitch, image_rows, pad, shuffle, flip, draw;
    int b;                    // Feistel half width: 4^b >= n, the least such b
    int vpr;                  // vectors per output row: W C_out / VEC
    int rpc, row_blocks;      // output rows per unit, units per image
    unsigned k0, k1, e0, e1;  // the key (seed lo, hi) and the epoch (lo, hi)
    unsigned short lut[4 * 256];   // bf16 bits of v(c, u) at [c][u]
};

constexpr int MIX_NONE = 0, MIX_MIXUP = 1, MIX_CUTMIX = 2;

// what the mixed batch adds: the partner's labels, the weights and box, and the fp32 values of the table (MixUp mixes those)
struct MixArgs : AugArgs {
    uint8_t *lab_b_out;       // [N] or NULL
    long long N;
    float lam, oml;           // RN32(lam), RN32(1 - lam), each formed in double
    int x1, y1, x2, y2;       // CutMix's box in output coordinates
    float flut[4 * 256];      // v(c, u) at [c][u]
};

template <int MODE>
using ArgsOf = typename std::conditional<MODE == MIX_NONE, AugArgs, MixArgs>::type;

// pi(e): a balanced Feistel network of FEISTEL_ROUNDS rounds over 2b bits, each round's function the low b bits of word x of the
// Philox block at counter (R, DOMAIN_AUG | DOMAIN_PERM | round, epoch lo, epoch hi), walked until the value is below n
__device__ unsigned long long permute(unsigned long long e, const AugArgs &a) {
    const unsigned mask = (1u << a.b) - 1u;
    unsigned long long v = e;
    do {
        unsigned L = (unsigned)(v >> a.b), R = (unsigned)v & mask;
#pragma unroll 1
        for (int r = 0; r < FEISTEL_ROUNDS; ++r) {
            const unsigned f = philox4x32_10(R, DOMAIN_AUG | DOMAIN_PERM | (unsigned)r, a.e0, a.e1, a.k0, a.k1).x & mask;
            const unsigned t = L ^ f;
            L = R;
            R = t;
        }
        v = ((unsigned long long)L << a.b) | R;
    } while (v >= (unsigned long long)a.n);
    return v;
}

template <int VEC>
struct alignas(2 * VEC) BitsVec {
    unsigned short h[VEC];
};

// the image at epoch position e and its crop and flip draws: dataset index i, oy, ox (offsets into the padded image) and flip
__device__ __forceinline__ void draw_unit(unsigned long long e, const AugArgs &a, unsigned long long &i, int &oy, int &ox, int &fl) {
    i = a.shuffle ? permute(e, a) : e;
    oy = 0, ox = 0, fl = 0;
    if (a.draw) {
        const uint4 w = philox4x32_10((unsigned)i, (unsigned)(i >> 32) | DOMAIN_AUG, a.e0, a.e1, a.k0, a.k1);
        const unsigned span = 2u * a.pad + 1u;
        oy = (int)__umulhi(w.x, span);
        ox = (int)__umulhi(w.y, span);
        fl = a.flip & (int)(w.z >> 31);
    }
}

// the source byte of output pixel (h, w), channel c, of an image drawn as (src, dy, dx, fl): 0 outside the image
__device__ __forceinline__ unsigned src_byte(const uint8_t *src, int h, int w, int c, int dy, int dx, int fl, const AugArgs &a) {
    const int sy = h + dy, sx = (fl ? a.W - 1 - w : w) + dx;
    return (unsigned)sy < (unsigned)a.H && (unsigned)sx < (unsigned)a.W ? __ldg(src + ((long long)sy * a.W + sx) * a.C + c) : 0u;
}

// x[j][h][w][c] = lut[c][src[i][h + oy - pad][w' + ox - pad][c]] (the byte 0 outside the image), w' = flip_i ? W - 1 - w : w;
// +0 for C <= c < C_out.  Pad columns and pad rows of x are never written.  MODE 1 (MixUp) writes
// bf16_rn(RN(RN(b * RN32(1 - lam)) + RN(a * RN32(lam)))) of the fp32 values a of j and b of its partner; MODE 2 (CutMix) the
// partner's element inside the box, j's outside.
template <int VEC, int MODE>
__global__ void __launch_bounds__(AUG_THREADS) k_augment(const __grid_constant__ ArgsOf<MODE> a) {
    __shared__ unsigned short lut[4 * 256];
    __shared__ float flut[4 * 256];                       // MixUp only
    __shared__ unsigned long long s_i, s_ib;
    __shared__ int s_oy, s_ox, s_fl, s_oyb, s_oxb, s_flb;
    for (int t = threadIdx.x; t < a.C * 256; t += AUG_THREADS) lut[t] = a.lut[t];
    if constexpr (MODE == MIX_MIXUP)
        for (int t = threadIdx.x; t < a.C * 256; t += AUG_THREADS) flut[t] = a.flut[t];
    for (long long u = blockIdx.x; u < a.units; u += gridDim.x) {
        const long long j = u / a.row_blocks;
        const int rb = (int)(u - j * a.row_blocks);
        if (threadIdx.x == 0) {
            unsigned long long i;
            int oy, ox, fl;
            draw_unit((unsigned long long)(a.first + j), a, i, oy, ox, fl);
            s_i = i;
            s_oy = oy - a.pad;
            s_ox = ox - a.pad;
            s_fl = fl;
            if (a.lab && rb == 0) a.lab_out[j] = a.lab[i];
        }
        if constexpr (MODE != MIX_NONE) {
            if (threadIdx.x == 32) {                          // the partner, beside thread 0 in a second warp
                const long long jb = j == 0 ? a.N - 1 : j - 1;
                unsigned long long i;
                int oy, ox, fl;
                draw_unit((unsigned long long)(a.first + jb), a, i, oy, ox, fl);
                s_ib = i;
                s_oyb = oy - a.pad;
                s_oxb = ox - a.pad;
                s_flb = fl;
                if (a.lab && rb == 0) a.lab_b_out[j] = a.lab[i];
            }
        }
        __syncthreads();
        const uint8_t *src = a.img + (long long)s_i * a.img_bytes;
        const int dy = s_oy, dx = s_ox, fl = s_fl;
        const int h0 = rb * a.rpc, rows = min(a.rpc, a.H - h0);
        __nv_bfloat16 *xj = a.x + j * a.image_rows * (long long)a.pitch;
        if constexpr (MODE == MIX_NONE) {
            const int WC = a.W * a.C;
            for (int t = threadIdx.x; t < rows * a.vpr; t += AUG_THREADS) {
                const int r = t / a.vpr;
                const int k = (t - r * a.vpr) * VEC;            // first element of the vector in its row
                const int h = h0 + r, sy = h + dy;
                const bool row_in = (unsigned)sy < (unsigned)a.H;
                const long long row_off = (long long)sy * WC;
                int w = k / a.C_out, c = k - w * a.C_out;
                BitsVec<VEC> out;
#pragma unroll
                for (int q = 0; q < VEC; ++q) {
                    unsigned short bits = 0;
                    if (c < a.C) {
                        const int sx = (fl ? a.W - 1 - w : w) + dx;
                        unsigned byte = 0;
                        if (row_in && (unsigned)sx < (unsigned)a.W) byte = __ldg(src + row_off + sx * a.C + c);
                        bits = lut[c * 256 + byte];
                    }
                    out.h[q] = bits;
                    if (++c == a.C_out) {
                        c = 0;
                        ++w;
                    }
                }
                *reinterpret_cast<BitsVec<VEC> *>(xj + (long long)h * a.pitch + k) = out;
            }
        } else {
            const uint8_t *srcb = a.img + (long long)s_ib * a.img_bytes;
            const int dyb = s_oyb, dxb = s_oxb, flb = s_flb;
            for (int t = threadIdx.x; t < rows * a.vpr; t += AUG_THREADS) {
                const int r = t / a.vpr;
                const int k = (t - r * a.vpr) * VEC;
                const int h = h0 + r;
                const bool row_box = h >= a.y1 && h < a.y2;
                int w = k / a.C_out, c = k - w * a.C_out;
                BitsVec<VEC> out;
#pragma unroll
                for (int q = 0; q < VEC; ++q) {
                    unsigned short bits = 0;
                    if (c < a.C) {
                        if constexpr (MODE == MIX_MIXUP) {
                            const float va = flut[c * 256 + src_byte(src, h, w, c, dy, dx, fl, a)];
                            const float vb = flut[c * 256 + src_byte(srcb, h, w, c, dyb, dxb, flb, a)];
                            bits = __bfloat16_as_ushort(__float2bfloat16_rn(__fadd_rn(__fmul_rn(vb, a.oml), __fmul_rn(va, a.lam))));
                        } else {
                            const bool p = row_box && w >= a.x1 && w < a.x2;
                            bits = lut[c * 256 + (p ? src_byte(srcb, h, w, c, dyb, dxb, flb, a) : src_byte(src, h, w, c, dy, dx, fl, a))];
                        }
                    }
                    out.h[q] = bits;
                    if (++c == a.C_out) {
                        c = 0;
                        ++w;
                    }
                }
                *reinterpret_cast<BitsVec<VEC> *>(xj + (long long)h * a.pitch + k) = out;
            }
        }
        __syncthreads();                                    // s_i .. s_flb are rewritten by the next unit
    }
}

// bf16 round to nearest even of an fp32 value, as __float2bfloat16_rn and torch's .to(bfloat16)
unsigned short bf16_rn(float f) {
    unsigned u;
    memcpy(&u, &f, 4);
    if ((u & 0x7FFFFFFFu) > 0x7F800000u) return 0x7FC0;
    u += 0x7FFFu + ((u >> 16) & 1u);
    return (unsigned short)(u >> 16);
}

// v(c, u): ToTensor, then Normalize's (t - mean) / std, each operation an fp32 round to nearest
float aug_value(const float *mean, const float *std_, int c, int u) {
    const float m = mean ? mean[c] : 0.0f, sd = std_ ? std_[c] : 1.0f;
    float v = (float)u / 255.0f;
    v = v - m;
    v = v / sd;
    return v;
}

struct AugShape {
    AugArgs a;
    int vec, grid;
};

// the domain, one message per rule, the table and the launch: a function of the arguments alone
int aug_shape(const char *fn, long long n, int H, int W, int C, long long first, int N, int shuffle, int pad, int flip, int C_out,
              int row_pitch, int image_rows, const float *mean, const float *std_, AugShape *s) {
    PCNN_REQUIRE(n >= 1 && N >= 1 && H >= 1 && W >= 1, PCNN_ERR_ARG, "%s: n = %lld, N = %d, H = %d, W = %d: each must be >= 1", fn, n,
                 N, H, W);
    PCNN_REQUIRE(first >= 0 && first <= n - N, PCNN_ERR_ARG, "%s: first = %lld, N = %d: 0 <= first and first + N <= n = %lld are required",
                 fn, first, N, n);
    PCNN_REQUIRE(C >= 1 && C <= 4, PCNN_ERR_ARG, "%s: C = %d: 1 <= C <= 4 is required", fn, C);
    PCNN_REQUIRE(C_out >= C && C_out <= 8, PCNN_ERR_ARG, "%s: C_out = %d: C = %d <= C_out <= 8 is required", fn, C_out, C);
    PCNN_REQUIRE(pad >= 0 && pad <= 64, PCNN_ERR_ARG, "%s: pad = %d: 0 <= pad <= 64 is required", fn, pad);
    PCNN_REQUIRE((shuffle == 0 || shuffle == 1) && (flip == 0 || flip == 1), PCNN_ERR_ARG,
                 "%s: shuffle = %d, flip = %d: each must be 0 or 1", fn, shuffle, flip);
    const long long img_bytes = (long long)H * W * C;
    PCNN_REQUIRE(img_bytes <= INT_MAX, PCNN_ERR_ARG, "%s: H W C = %lld: one image must fit the 32-bit range (< 2^31 bytes)", fn,
                 img_bytes);
    PCNN_REQUIRE(n <= ((1LL << 62) - 1) / img_bytes, PCNN_ERR_ARG, "%s: n H W C = %lld x %lld: the dataset must be below 2^62 bytes", fn,
                 n, img_bytes);
    const long long row_elems = (long long)W * C_out, dense = (row_elems + 7) / 8 * 8;
    const long long pitch = row_pitch == 0 ? dense : row_pitch;
    PCNN_REQUIRE(pitch >= row_elems && pitch % 8 == 0 && pitch <= INT_MAX, PCNN_ERR_ARG,
                 "%s: row_pitch = %d: 0 (W C_out = %lld rounded up to 8) or a multiple of 8 >= W C_out is required", fn, row_pitch,
                 row_elems);
    const int rows = image_rows == 0 ? H : image_rows;
    PCNN_REQUIRE(rows >= H, PCNN_ERR_ARG, "%s: image_rows = %d: 0 (H) or >= H = %d is required", fn, image_rows, H);
    PCNN_REQUIRE((double)N * rows * (double)pitch * 2.0 < 4611686018427387904.0, PCNN_ERR_ARG,
                 "%s: N image_rows row_pitch = %d x %d x %lld: x must be below 2^62 bytes", fn, N, rows, pitch);
    for (int c = 0; c < C; ++c)
        PCNN_REQUIRE(!mean || std::isfinite(mean[c]), PCNN_ERR_ARG, "%s: mean[%d] = %g: a finite mean is required", fn, c,
                     mean ? (double)mean[c] : 0.0);
    for (int c = 0; c < C; ++c)
        PCNN_REQUIRE(!std_ || (std::isfinite(std_[c]) && std_[c] > 0.0f), PCNN_ERR_ARG, "%s: std[%d] = %g: a finite std > 0 is required",
                     fn, c, std_ ? (double)std_[c] : 1.0);
    AugArgs &a = s->a;
    memset(&a, 0, sizeof(a));
    a.n = n;
    a.first = first;
    a.img_bytes = img_bytes;
    a.H = H;
    a.W = W;
    a.C = C;
    a.C_out = C_out;
    a.pitch = (int)pitch;
    a.image_rows = rows;
    a.pad = pad;
    a.shuffle = shuffle;
    a.flip = flip;
    a.draw = pad > 0 || flip;
    a.b = 0;
    while ((1ULL << (2 * a.b)) < (unsigned long long)n) ++a.b;
    s->vec = row_elems % 8 == 0 ? 8 : 1;
    a.vpr = (int)(row_elems / s->vec);
    a.rpc = (int)std::min<long long>(H, std::max<long long>(1, (AUG_CTA_BYTES + row_elems * 2 - 1) / (row_elems * 2)));
    a.row_blocks = (H + a.rpc - 1) / a.rpc;
    a.units = (long long)N * a.row_blocks;
    s->grid = (int)std::min(AUG_MAX_GRID, a.units);
    for (int c = 0; c < C; ++c)
        for (int u = 0; u < 256; ++u) a.lut[c * 256 + u] = bf16_rn(aug_value(mean, std_, c, u));
    return PCNN_OK;
}

bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

bool disjoint(const void *a, size_t abytes, const void *b, size_t bbytes) {
    if (!a || !b) return true;
    const uintptr_t pa = (uintptr_t)a, pb = (uintptr_t)b;
    return pa + abytes <= pb || pb + bbytes <= pa;
}

}  // namespace

extern "C" int pcnn_augment_u8_bf16_info(long long n, int H, int W, int C, long long first, int N, int shuffle, int pad, int flip,
                                         int C_out, int row_pitch, int image_rows, const float *mean_host, const float *std_host,
                                         long long *out8, uint16_t *lut_out) {
    const char *fn = "pcnn_augment_u8_bf16_info";
    PCNN_REQUIRE(out8, PCNN_ERR_ARG, "%s: NULL out8", fn);
    AugShape s;
    const int rc = aug_shape(fn, n, H, W, C, first, N, shuffle, pad, flip, C_out, row_pitch, image_rows, mean_host, std_host, &s);
    if (rc) return rc;
    out8[0] = s.a.pitch;
    out8[1] = s.a.image_rows;
    out8[2] = s.a.b;
    out8[3] = s.vec;
    out8[4] = s.grid;
    out8[5] = s.a.rpc;
    out8[6] = s.a.row_blocks;
    out8[7] = AUG_THREADS;
    if (lut_out) memcpy(lut_out, s.a.lut, sizeof(uint16_t) * 256 * C);
    return PCNN_OK;
}

// the plain call's checks, one message per rule, and its arguments: everything but the launch
int aug_prepare(const char *fn, pcnn_ctx *ctx, const uint8_t *images_dev, const uint8_t *labels_dev, long long n, int H, int W, int C,
                long long first, int N, int shuffle, int pad, int flip, unsigned long long seed, unsigned long long epoch,
                const float *mean_host, const float *std_host, void *x_bf16_dev, int C_out, int row_pitch, int image_rows,
                uint8_t *labels_out_dev, AugShape *s, size_t *xbytes_out) {
    PCNN_REQUIRE(ctx && images_dev && x_bf16_dev, PCNN_ERR_ARG, "%s: NULL context, images or x (only the labels may be NULL)", fn);
    PCNN_REQUIRE(!labels_dev == !labels_out_dev, PCNN_ERR_ARG, "%s: labels and labels_out must both be NULL or neither", fn);
    const int rc = aug_shape(fn, n, H, W, C, first, N, shuffle, pad, flip, C_out, row_pitch, image_rows, mean_host, std_host, s);
    if (rc) return rc;
    PCNN_REQUIRE(aligned16(x_bf16_dev), PCNN_ERR_ARG, "%s: x must be 16-byte aligned", fn);
    const size_t xbytes = (((size_t)N - 1) * s->a.image_rows * s->a.pitch + (size_t)(H - 1) * s->a.pitch + (size_t)W * C_out) * 2;
    PCNN_REQUIRE(disjoint(x_bf16_dev, xbytes, images_dev, (size_t)n * s->a.img_bytes) && disjoint(x_bf16_dev, xbytes, labels_out_dev, N),
                 PCNN_ERR_ARG, "%s: overlapping buffers: x must share no byte with images or labels_out", fn);
    PCNN_REQUIRE(disjoint(labels_out_dev, N, labels_dev, n) && disjoint(labels_out_dev, N, images_dev, (size_t)n * s->a.img_bytes),
                 PCNN_ERR_ARG, "%s: overlapping buffers: labels_out must share no byte with labels or images", fn);
    AugArgs &a = s->a;
    a.img = images_dev;
    a.lab = labels_dev;
    a.x = static_cast<__nv_bfloat16 *>(x_bf16_dev);
    a.lab_out = labels_out_dev;
    a.k0 = (unsigned)seed;
    a.k1 = (unsigned)(seed >> 32);
    a.e0 = (unsigned)epoch;
    a.e1 = (unsigned)(epoch >> 32);
    *xbytes_out = xbytes;
    return PCNN_OK;
}

extern "C" int pcnn_augment_u8_bf16(pcnn_ctx *ctx, const uint8_t *images_dev, const uint8_t *labels_dev, long long n, int H, int W, int C,
                                    long long first, int N, int shuffle, int pad, int flip, unsigned long long seed,
                                    unsigned long long epoch, const float *mean_host, const float *std_host, void *x_bf16_dev, int C_out,
                                    int row_pitch, int image_rows, uint8_t *labels_out_dev) {
    AugShape s;
    size_t xbytes;
    const int rc = aug_prepare("pcnn_augment_u8_bf16", ctx, images_dev, labels_dev, n, H, W, C, first, N, shuffle, pad, flip, seed, epoch,
                               mean_host, std_host, x_bf16_dev, C_out, row_pitch, image_rows, labels_out_dev, &s, &xbytes);
    if (rc) return rc;
    pcnn_device_guard dg(ctx->device);
    if (s.vec == 8)
        k_augment<8, MIX_NONE><<<s.grid, AUG_THREADS, 0, ctx->stream>>>(s.a);
    else
        k_augment<1, MIX_NONE><<<s.grid, AUG_THREADS, 0, ctx->stream>>>(s.a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_augment_mix_u8_bf16(pcnn_ctx *ctx, const uint8_t *images_dev, const uint8_t *labels_dev, long long n, int H, int W,
                                        int C, long long first, int N, int shuffle, int pad, int flip, unsigned long long seed,
                                        unsigned long long epoch, const float *mean_host, const float *std_host, void *x_bf16_dev,
                                        int C_out, int row_pitch, int image_rows, uint8_t *labels_out_dev, int mode, double lam, int x1,
                                        int y1, int x2, int y2, uint8_t *labels_b_out_dev) {
    const char *fn = "pcnn_augment_mix_u8_bf16";
    AugShape s;
    size_t xbytes;
    const int rc = aug_prepare(fn, ctx, images_dev, labels_dev, n, H, W, C, first, N, shuffle, pad, flip, seed, epoch, mean_host, std_host,
                               x_bf16_dev, C_out, row_pitch, image_rows, labels_out_dev, &s, &xbytes);
    if (rc) return rc;
    PCNN_REQUIRE(mode == MIX_MIXUP || mode == MIX_CUTMIX, PCNN_ERR_ARG, "%s: mode = %d: 1 (MixUp) or 2 (CutMix) is required", fn, mode);
    PCNN_REQUIRE(std::isfinite(lam) && lam >= 0.0 && lam <= 1.0, PCNN_ERR_ARG, "%s: lam = %g: a finite 0 <= lam <= 1 is required", fn, lam);
    PCNN_REQUIRE(x1 >= 0 && x1 <= x2 && x2 <= W, PCNN_ERR_ARG, "%s: x1 = %d, x2 = %d: 0 <= x1 <= x2 <= W = %d is required", fn, x1, x2, W);
    PCNN_REQUIRE(y1 >= 0 && y1 <= y2 && y2 <= H, PCNN_ERR_ARG, "%s: y1 = %d, y2 = %d: 0 <= y1 <= y2 <= H = %d is required", fn, y1, y2, H);
    PCNN_REQUIRE(!labels_dev == !labels_b_out_dev, PCNN_ERR_ARG, "%s: labels and labels_b_out must both be NULL or neither", fn);
    PCNN_REQUIRE(disjoint(labels_b_out_dev, N, x_bf16_dev, xbytes) && disjoint(labels_b_out_dev, N, images_dev, (size_t)n * s.a.img_bytes) &&
                     disjoint(labels_b_out_dev, N, labels_dev, n) && disjoint(labels_b_out_dev, N, labels_out_dev, N),
                 PCNN_ERR_ARG, "%s: overlapping buffers: labels_b_out must share no byte with x, images, labels or labels_out", fn);
    MixArgs m{};
    static_cast<AugArgs &>(m) = s.a;
    m.lab_b_out = labels_b_out_dev;
    m.N = N;
    m.lam = (float)lam;
    m.oml = (float)(1.0 - lam);
    m.x1 = x1;
    m.y1 = y1;
    m.x2 = x2;
    m.y2 = y2;
    for (int c = 0; c < C; ++c)
        for (int u = 0; u < 256; ++u) m.flut[c * 256 + u] = aug_value(mean_host, std_host, c, u);
    pcnn_device_guard dg(ctx->device);
    if (mode == MIX_MIXUP) {
        if (s.vec == 8)
            k_augment<8, MIX_MIXUP><<<s.grid, AUG_THREADS, 0, ctx->stream>>>(m);
        else
            k_augment<1, MIX_MIXUP><<<s.grid, AUG_THREADS, 0, ctx->stream>>>(m);
    } else {
        if (s.vec == 8)
            k_augment<8, MIX_CUTMIX><<<s.grid, AUG_THREADS, 0, ctx->stream>>>(m);
        else
            k_augment<1, MIX_CUTMIX><<<s.grid, AUG_THREADS, 0, ctx->stream>>>(m);
    }
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
