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
#include <memory>
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

int aug_launch(pcnn_ctx *ctx, const AugShape &s) {
    if (s.vec == 8)
        k_augment<8, MIX_NONE><<<s.grid, AUG_THREADS, 0, ctx->stream>>>(s.a);
    else
        k_augment<1, MIX_NONE><<<s.grid, AUG_THREADS, 0, ctx->stream>>>(s.a);
    PCNN_CHECK_LAUNCH(ctx);
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
    return aug_launch(ctx, s);
}

// ------------------------------------------------------------------------------------------------ segmentation masks
// pcnn_augment_mask_u8: the uint8 masks [n][H][W] of the plain call's batch, each moved exactly as its image: position e of the
// epoch takes mask pi(e) with the crop and flip of draw_unit, the same Philox block the image kernel reads.  One CTA per batch
// position; the padding reads fill.
namespace {

__global__ void __launch_bounds__(AUG_THREADS) k_augment_mask(const __grid_constant__ AugArgs a, const uint8_t *__restrict__ masks,
                                                              uint8_t *__restrict__ out, long long N, int fill) {
    __shared__ unsigned long long s_i;
    __shared__ int s_oy, s_ox, s_fl;
    const int hw = a.H * a.W;
    for (long long j = blockIdx.x; j < N; j += gridDim.x) {
        if (threadIdx.x == 0) {
            unsigned long long i;
            int oy, ox, fl;
            draw_unit((unsigned long long)(a.first + j), a, i, oy, ox, fl);
            s_i = i;
            s_oy = oy - a.pad;
            s_ox = ox - a.pad;
            s_fl = fl;
        }
        __syncthreads();
        const uint8_t *src = masks + (long long)s_i * hw;
        for (int p = threadIdx.x; p < hw; p += AUG_THREADS) {
            const int h = p / a.W, w = p - h * a.W;
            const int sy = h + s_oy, sx = (s_fl ? a.W - 1 - w : w) + s_ox;
            out[j * hw + p] = (unsigned)sy < (unsigned)a.H && (unsigned)sx < (unsigned)a.W ? __ldg(src + (long long)sy * a.W + sx)
                                                                                            : (uint8_t)fill;
        }
        __syncthreads();                                    // s_i .. s_fl are rewritten by the next position
    }
}

}  // namespace

extern "C" int pcnn_augment_mask_u8(pcnn_ctx *ctx, const uint8_t *masks_dev, long long n, int H, int W, long long first, int N, int shuffle,
                                    int pad, int flip, unsigned long long seed, unsigned long long epoch, int mask_fill,
                                    uint8_t *masks_out_dev) {
    const char *fn = "pcnn_augment_mask_u8";
    PCNN_REQUIRE(ctx && masks_dev && masks_out_dev, PCNN_ERR_ARG, "%s: NULL context, masks or masks_out", fn);
    PCNN_REQUIRE(mask_fill >= 0 && mask_fill <= 255, PCNN_ERR_ARG, "%s: mask_fill = %d: 0 .. 255 is required", fn, mask_fill);
    AugShape s;
    const int rc = aug_shape(fn, n, H, W, 1, first, N, shuffle, pad, flip, 1, 0, 0, nullptr, nullptr, &s);
    if (rc) return rc;
    PCNN_REQUIRE(disjoint(masks_out_dev, (size_t)N * H * W, masks_dev, (size_t)n * H * W), PCNN_ERR_ARG,
                 "%s: overlapping buffers: masks_out must share no byte with masks", fn);
    AugArgs &a = s.a;
    a.k0 = (unsigned)seed;
    a.k1 = (unsigned)(seed >> 32);
    a.e0 = (unsigned)epoch;
    a.e1 = (unsigned)(epoch >> 32);
    pcnn_device_guard dg(ctx->device);
    const int grid = (int)std::min<long long>(AUG_MAX_GRID, N);
    k_augment_mask<<<grid, AUG_THREADS, 0, ctx->stream>>>(a, masks_dev, masks_out_dev, N, mask_fill);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

// ------------------------------------------------------------------------------------------------ resized batches
// pcnn_augment_resized_u8_bf16: RandomResizedCrop (mode 1) or Resize + CenterCrop (mode 2) by torch's uint8 antialiased bilinear
// resample, the fixed-point separable rule include/pcnn.h states.  A CTA takes one (batch position, block of output rows) unit:
// thread 0 walks the permutation and draws the box; the CTA finds each axis' largest weight (it sets the fixed-point precision),
// forms the int16 taps of the window's columns and of its own rows in shared memory, runs the horizontal pass over only the source
// rows those rows reach into a uint8 intermediate in shared memory, then the vertical pass, the flip and the table lookup.
namespace {

constexpr int RES_TRAIN = 1, RES_EVAL = 2;
constexpr int RES_MAX_TAPS = 33;              // 2 ceil(support) + 1 per axis: a downscale of at most 16x
constexpr int RES_MAX_SIDE = 16384;           // output, resized and resize sides: each CTA walks a whole axis for its largest weight
constexpr int RES_MAX_RPC = 32;               // output rows per unit
constexpr int RES_SMEM_LIMIT = 48 * 1024;     // static + dynamic shared memory of a CTA: the limit that needs no opt-in
constexpr unsigned DOMAIN_BOX = 0xC0000000u;  // counter word 1 of box block k: DOMAIN_BOX | (8 + k) << 24 | i hi, i < 2^56
constexpr int BOX_ATTEMPTS = 10;

struct ResArgs : AugArgs {
    int mode, H_out, W_out;
    int Rh, Rw, ty, tx;                     // the resized image and the window's offset in it (mode 1: H_out, W_out, 0, 0)
    int fb_top, fb_left, fb_h, fb_w;        // torchvision's central fallback crop
    float s0, srange, lr0, lrange;          // RN32(s0), RN32(RN32(s1) - RN32(s0)), RN32(log r0), RN32(RN32(log r1) - RN32(log r0))
    int taps_y, taps_x, rows_cap;           // worst-case taps per axis; source rows of one unit's intermediate
    int off_y0, off_wx, off_wy, off_mid;    // byte offsets in dynamic shared memory: y0 / yn, wx, wy, the intermediate
};

// image i's box (top, left, height, width) in source pixels: torchvision's RandomResizedCrop.get_params on Philox draws
__device__ void draw_box(unsigned long long i, const ResArgs &a, int &top, int &left, int &bh, int &bw) {
    const unsigned lo = (unsigned)i, hi = (unsigned)(i >> 32);
    const double area = __dmul_rn((double)a.H, (double)a.W);
    uint4 w = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 1
    for (int t = 0; t < BOX_ATTEMPTS; ++t) {
        if ((t & 1) == 0) w = philox4x32_10(lo, DOMAIN_BOX | (unsigned)(8 + t / 2) << 24 | hi, a.e0, a.e1, a.k0, a.k1);
        const unsigned us = (t & 1) ? w.z : w.x, ul = (t & 1) ? w.w : w.y;
        const float s = __fadd_rn(__fmul_rn(__fmul_rn((float)(us >> 8), 5.96046448e-08f), a.srange), a.s0);
        const float lr = __fadd_rn(__fmul_rn(__fmul_rn((float)(ul >> 8), 5.96046448e-08f), a.lrange), a.lr0);
        const double aspect = (double)exp_f32(lr), ta = __dmul_rn(area, (double)s);
        const double cw = rint(__dsqrt_rn(__dmul_rn(ta, aspect))), ch = rint(__dsqrt_rn(__ddiv_rn(ta, aspect)));
        if (cw > 0.0 && cw <= (double)a.W && ch > 0.0 && ch <= (double)a.H) {
            bw = (int)cw;
            bh = (int)ch;
            const uint4 r = philox4x32_10(lo, DOMAIN_BOX | (unsigned)(8 + BOX_ATTEMPTS / 2) << 24 | hi, a.e0, a.e1, a.k0, a.k1);
            top = (int)__umulhi(r.x, (unsigned)(a.H - bh + 1));
            left = (int)__umulhi(r.y, (unsigned)(a.W - bw + 1));
            return;
        }
    }
    top = a.fb_top, left = a.fb_left, bh = a.fb_h, bw = a.fb_w;
}

// one axis of the resample, in -> out pixels; every double operation rounded on its own (no contraction)
struct Axis {
    double scale, support, invscale;
    int in, taps;
    __device__ Axis(int in_, int out) : in(in_) {
        scale = __ddiv_rn((double)in_, (double)out);
        support = scale >= 1.0 ? scale : 1.0;
        invscale = scale >= 1.0 ? __ddiv_rn(1.0, scale) : 1.0;
        taps = (int)ceil(support) * 2 + 1;
    }
    // the first tap and the tap count of output coordinate o, and its centre
    __device__ __forceinline__ int range(int o, int &xmin, double &center) const {
        center = __dmul_rn(scale, __dadd_rn((double)o, 0.5));
        xmin = max((int)(long long)__dadd_rn(__dsub_rn(center, support), 0.5), 0);
        const int xmax = (int)min((long long)__dadd_rn(__dadd_rn(center, support), 0.5), (long long)in);
        return min(max(xmax - xmin, 0), taps);
    }
    // the unnormalised weight of tap j
    __device__ __forceinline__ double weight(int j, int xmin, double center) const {
        const double x = fabs(__dmul_rn(__dadd_rn(__dsub_rn((double)(j + xmin), center), 0.5), invscale));
        return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
    }
    __device__ __forceinline__ double total(int n, int xmin, double center) const {
        double t = 0.0;
        for (int j = 0; j < n; ++j) t = __dadd_rn(t, weight(j, xmin, center));
        return t;
    }
    // the largest normalised weight of coordinate o
    __device__ double wmax(int o) const {
        int xmin;
        double c;
        const int n = range(o, xmin, c);
        const double t = total(n, xmin, c);
        double m = 0.0;
        if (t != 0.0)
            for (int j = 0; j < n; ++j) m = fmax(m, __ddiv_rn(weight(j, xmin, c), t));
        return m;
    }
    // coordinate o's taps as int16 at 2^prec (taps past the count are 0); returns the count, xmin through the reference
    __device__ int quantise(int o, int prec, int &xmin, short *q, int stride) const {
        double c;
        const int n = range(o, xmin, c);
        const double t = total(n, xmin, c), one = (double)(1 << prec);
        for (int j = 0; j < stride; ++j) {
            const double w = j < n && t != 0.0 ? __ddiv_rn(weight(j, xmin, c), t) : 0.0;
            q[j] = (short)(int)__dadd_rn(__dmul_rn(w, one), 0.5);       // w >= 0
        }
        return n;
    }
};

// the precision of an axis whose largest weight is m: the largest p <= 22 below the first whose next step reaches 2^15
__device__ __forceinline__ int precision(double m) {
    int p = 0;
    for (; p < 22; ++p)
        if ((int)__dadd_rn(0.5, __dmul_rn(m, (double)(1 << (p + 1)))) >= (1 << 15)) break;
    return p;
}

__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// the kernel's static shared memory, one object so that the host can budget the dynamic part as RES_SMEM_LIMIT minus its size
struct ResShared {
    unsigned short lut[4 * 256];
    unsigned long long i;
    int top, left, bh, bw, fl, px, py, lo, hi;
    double my[AUG_THREADS / 32], mx[AUG_THREADS / 32];
};
// a block's static plus dynamic shared memory must fit the 48 KB a launch gets without an opt-in; the dynamic part starts 16-byte
// aligned after the static object
constexpr int RES_SMEM = RES_SMEM_LIMIT - (int)((sizeof(ResShared) + 15) / 16 * 16);

template <int VEC>
__global__ void __launch_bounds__(AUG_THREADS) k_augment_resized(const __grid_constant__ ResArgs a) {
    __shared__ ResShared sh;
    extern __shared__ __align__(16) unsigned char smem[];
    int *x0 = reinterpret_cast<int *>(smem), *xn = x0 + a.W_out;                 // source column of tap 0 (-1: fill), tap count
    int *y0 = reinterpret_cast<int *>(smem + a.off_y0), *yn = y0 + a.rpc;       // box row of tap 0, tap count
    short *wx = reinterpret_cast<short *>(smem + a.off_wx), *wy = reinterpret_cast<short *>(smem + a.off_wy);
    uint8_t *mid = smem + a.off_mid;                                             // [rows][W_out][C]
    for (int t = threadIdx.x; t < a.C * 256; t += AUG_THREADS) sh.lut[t] = a.lut[t];
    const int RWC = a.W_out * a.C;
    for (long long u = blockIdx.x; u < a.units; u += gridDim.x) {
        const long long j = u / a.row_blocks;
        const int rb = (int)(u - j * a.row_blocks);
        if (threadIdx.x == 0) {
            const unsigned long long e = (unsigned long long)(a.first + j);
            const unsigned long long i = a.shuffle ? permute(e, a) : e;
            int top = 0, left = 0, bh = a.H, bw = a.W;
            if (a.mode == RES_TRAIN) draw_box(i, a, top, left, bh, bw);
            sh.i = i;
            sh.top = top, sh.left = left, sh.bh = bh, sh.bw = bw;
            sh.fl = a.flip ? (int)(philox4x32_10((unsigned)i, (unsigned)(i >> 32) | DOMAIN_AUG, a.e0, a.e1, a.k0, a.k1).z >> 31) : 0;
            if (a.lab && rb == 0) a.lab_out[j] = a.lab[i];
        }
        __syncthreads();
        const Axis ay(sh.bh, a.Rh), ax(sh.bw, a.Rw);
        double my = 0.0, mx = 0.0;
        for (int t = threadIdx.x; t < a.Rh + a.Rw; t += AUG_THREADS) {
            if (t < a.Rh) my = fmax(my, ay.wmax(t));
            else mx = fmax(mx, ax.wmax(t - a.Rh));
        }
        my = warp_max(my);
        mx = warp_max(mx);
        if ((threadIdx.x & 31) == 0) sh.my[threadIdx.x >> 5] = my, sh.mx[threadIdx.x >> 5] = mx;
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int k = 1; k < AUG_THREADS / 32; ++k) my = fmax(my, sh.my[k]), mx = fmax(mx, sh.mx[k]);
            sh.py = precision(fmax(my, sh.my[0]));
            sh.px = precision(fmax(mx, sh.mx[0]));
        }
        __syncthreads();
        const int py = sh.py, px = sh.px, h0 = rb * a.rpc, rows = min(a.rpc, a.H_out - h0);
        for (int t = threadIdx.x; t < a.W_out + rows; t += AUG_THREADS) {
            if (t < a.W_out) {
                const int rx = t + a.tx;
                int xmin = 0;
                xn[t] = rx >= 0 && rx < a.Rw ? ax.quantise(rx, px, xmin, wx + t * a.taps_x, a.taps_x) : 0;
                x0[t] = rx >= 0 && rx < a.Rw ? sh.left + xmin : -1;
            } else {
                const int r = t - a.W_out, ry = h0 + r + a.ty;
                int ymin = 0;
                yn[r] = ry >= 0 && ry < a.Rh ? ay.quantise(ry, py, ymin, wy + r * a.taps_y, a.taps_y) : 0;
                y0[r] = ry >= 0 && ry < a.Rh ? ymin : -1;
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int lo = INT_MAX, hi = 0;
            for (int r = 0; r < rows; ++r)
                if (y0[r] >= 0) lo = min(lo, y0[r]), hi = max(hi, y0[r] + yn[r]);
            sh.lo = lo == INT_MAX ? 0 : lo;                     // no row in the resized image (eval): an empty pass
            sh.hi = lo == INT_MAX ? 0 : hi;
        }
        __syncthreads();
        const int lo = sh.lo, nmid = sh.hi - sh.lo;                // 0 <= nmid <= rows_cap
        const uint8_t *src = a.img + (long long)sh.i * a.img_bytes + ((long long)(sh.top + lo) * a.W) * a.C;
        for (int t = threadIdx.x; t < nmid * RWC; t += AUG_THREADS) {
            const int r = t / RWC, k = t - r * RWC, x = k / a.C, c = k - x * a.C;
            if (x0[x] < 0) continue;
            const uint8_t *p = src + ((long long)r * a.W + x0[x]) * a.C + c;
            const short *w = wx + x * a.taps_x;
            int acc = 1 << (px - 1);
            for (int q = 0; q < xn[x]; ++q) acc += (int)__ldg(p + q * a.C) * w[q];
            mid[t] = (uint8_t)min(max(acc >> px, 0), 255);
        }
        __syncthreads();
        const int fl = sh.fl;
        __nv_bfloat16 *xj = a.x + j * a.image_rows * (long long)a.pitch;
        for (int t = threadIdx.x; t < rows * a.vpr; t += AUG_THREADS) {
            const int r = t / a.vpr;
            const int k = (t - r * a.vpr) * VEC;
            const bool row_in = y0[r] >= 0;
            const uint8_t *m = mid + (row_in ? y0[r] - lo : 0) * RWC;
            const short *w = wy + r * a.taps_y;
            int ow = k / a.C_out, c = k - ow * a.C_out;
            BitsVec<VEC> out;
#pragma unroll
            for (int q = 0; q < VEC; ++q) {
                unsigned short bits = 0;
                if (c < a.C) {
                    const int x = fl ? a.W_out - 1 - ow : ow;
                    unsigned byte = 0;
                    if (row_in && x0[x] >= 0) {
                        int acc = 1 << (py - 1);
                        for (int p = 0; p < yn[r]; ++p) acc += (int)m[p * RWC + x * a.C + c] * w[p];
                        byte = (unsigned)min(max(acc >> py, 0), 255);
                    }
                    bits = sh.lut[c * 256 + byte];
                }
                out.h[q] = bits;
                if (++c == a.C_out) {
                    c = 0;
                    ++ow;
                }
            }
            *reinterpret_cast<BitsVec<VEC> *>(xj + (long long)(h0 + r) * a.pitch + k) = out;
        }
        __syncthreads();                                          // the shared state is rewritten by the next unit
    }
}

struct ResShape {
    ResArgs a;
    int vec, grid, smem;
};

long long round_half_even(double v) { return (long long)std::nearbyint(v); }

// worst-case taps of an axis: the whole image, in pixels, resampled to out
int worst_taps(int in, int out) { return (int)std::ceil(std::max((double)in / out, 1.0)) * 2 + 1; }

// source rows a unit of rpc output rows can reach on an in -> out axis, plus one of slack for rounding
int rows_cap(int in, int out, int rpc) {
    const double scale = (double)in / out, support = std::max(scale, 1.0);
    return (int)std::min<double>(in, std::floor(scale * (rpc - 1) + 2.0 * support + 1.0) + 2.0);
}

// dynamic shared memory of a unit of rpc rows whose intermediate holds cap source rows; sets the offsets of its parts (16-byte
// aligned): x0 / xn, y0 / yn, wx, wy, the intermediate
long long res_smem(ResArgs &a, int rpc, int cap) {
    auto up = [](long long v) { return (v + 15) / 16 * 16; };
    const long long y0 = up(8LL * a.W_out), wx = y0 + up(8LL * rpc), wy = wx + up(2LL * a.W_out * a.taps_x),
                    mid = wy + up(2LL * rpc * a.taps_y);
    a.off_y0 = (int)y0, a.off_wx = (int)wx, a.off_wy = (int)wy, a.off_mid = (int)mid;
    return mid + (long long)cap * a.W_out * a.C;
}

// the domain, one message per rule, the table, the boxes' constants and the launch: a function of the arguments alone
int res_shape(const char *fn, long long n, int H, int W, int C, long long first, int N, int shuffle, int flip, int H_out, int W_out,
              int C_out, int row_pitch, int image_rows, const float *mean, const float *std_, int mode, double s0, double s1, double r0,
              double r1, int resize_size, ResShape *s) {
    PCNN_REQUIRE(n >= 1 && N >= 1 && H >= 1 && W >= 1 && H_out >= 1 && W_out >= 1, PCNN_ERR_ARG,
                 "%s: n = %lld, N = %d, H = %d, W = %d, H_out = %d, W_out = %d: each must be >= 1", fn, n, N, H, W, H_out, W_out);
    PCNN_REQUIRE(first >= 0 && first <= n - N, PCNN_ERR_ARG, "%s: first = %lld, N = %d: 0 <= first and first + N <= n = %lld are required",
                 fn, first, N, n);
    PCNN_REQUIRE(n <= (1LL << 56), PCNN_ERR_ARG, "%s: n = %lld: n <= 2^56 is required (the box counters hold the index in 56 bits)", fn, n);
    PCNN_REQUIRE(C >= 1 && C <= 4, PCNN_ERR_ARG, "%s: C = %d: 1 <= C <= 4 is required", fn, C);
    PCNN_REQUIRE(C_out >= C && C_out <= 8, PCNN_ERR_ARG, "%s: C_out = %d: C = %d <= C_out <= 8 is required", fn, C_out, C);
    PCNN_REQUIRE((shuffle == 0 || shuffle == 1) && (flip == 0 || flip == 1), PCNN_ERR_ARG,
                 "%s: shuffle = %d, flip = %d: each must be 0 or 1", fn, shuffle, flip);
    PCNN_REQUIRE(mode == RES_TRAIN || mode == RES_EVAL, PCNN_ERR_ARG, "%s: mode = %d: 1 (train) or 2 (eval) is required", fn, mode);
    const long long img_bytes = (long long)H * W * C;
    PCNN_REQUIRE(img_bytes <= INT_MAX, PCNN_ERR_ARG, "%s: H W C = %lld: one image must fit the 32-bit range (< 2^31 bytes)", fn,
                 img_bytes);
    PCNN_REQUIRE(n <= ((1LL << 62) - 1) / img_bytes, PCNN_ERR_ARG, "%s: n H W C = %lld x %lld: the dataset must be below 2^62 bytes", fn,
                 n, img_bytes);
    PCNN_REQUIRE(H_out <= RES_MAX_SIDE && W_out <= RES_MAX_SIDE, PCNN_ERR_ARG, "%s: H_out = %d, W_out = %d: each must be <= %d", fn,
                 H_out, W_out, RES_MAX_SIDE);
    const long long row_elems = (long long)W_out * C_out, dense = (row_elems + 7) / 8 * 8;
    const long long pitch = row_pitch == 0 ? dense : row_pitch;
    PCNN_REQUIRE(pitch >= row_elems && pitch % 8 == 0 && pitch <= INT_MAX, PCNN_ERR_ARG,
                 "%s: row_pitch = %d: 0 (W_out C_out = %lld rounded up to 8) or a multiple of 8 >= W_out C_out is required", fn,
                 row_pitch, row_elems);
    const int rows = image_rows == 0 ? H_out : image_rows;
    PCNN_REQUIRE(rows >= H_out, PCNN_ERR_ARG, "%s: image_rows = %d: 0 (H_out) or >= H_out = %d is required", fn, image_rows, H_out);
    PCNN_REQUIRE((double)N * rows * (double)pitch * 2.0 < 4611686018427387904.0, PCNN_ERR_ARG,
                 "%s: N image_rows row_pitch = %d x %d x %lld: x must be below 2^62 bytes", fn, N, rows, pitch);
    for (int c = 0; c < C; ++c)
        PCNN_REQUIRE(!mean || std::isfinite(mean[c]), PCNN_ERR_ARG, "%s: mean[%d] = %g: a finite mean is required", fn, c,
                     mean ? (double)mean[c] : 0.0);
    for (int c = 0; c < C; ++c)
        PCNN_REQUIRE(!std_ || (std::isfinite(std_[c]) && std_[c] > 0.0f), PCNN_ERR_ARG, "%s: std[%d] = %g: a finite std > 0 is required",
                     fn, c, std_ ? (double)std_[c] : 1.0);
    ResArgs &a = s->a;
    memset(&a, 0, sizeof(a));
    if (mode == RES_TRAIN) {
        const double lo = 1.1754943508222875e-38, hi = 3.4028234663852886e+38;   // fp32's normal range
        auto normal = [&](double v) { return v >= lo && v <= hi; };
        PCNN_REQUIRE(normal(s0) && normal(s1) && normal(r0) && normal(r1), PCNN_ERR_ARG,
                     "%s: scale = (%g, %g), ratio = (%g, %g): each must be finite and within fp32's normal range [2^-126, 3.4028235e38]",
                     fn, s0, s1, r0, r1);
        PCNN_REQUIRE(s0 <= s1 && r0 <= r1, PCNN_ERR_ARG, "%s: scale = (%g, %g), ratio = (%g, %g): each range must be (min, max)", fn,
                     s0, s1, r0, r1);
        const double in_ratio = (double)W / (double)H;
        int fh = H, fw = W;
        if (in_ratio < r0)
            fh = (int)round_half_even(fw / r0);
        else if (in_ratio > r1)
            fw = (int)round_half_even(fh * r1);
        PCNN_REQUIRE(fh >= 1 && fw >= 1, PCNN_ERR_ARG, "%s: ratio = (%g, %g): the central fallback crop of a %d x %d image is empty", fn,
                     r0, r1, H, W);
        a.fb_h = fh, a.fb_w = fw, a.fb_top = (H - fh) / 2, a.fb_left = (W - fw) / 2;
        const float s0f = (float)s0, s1f = (float)s1, l0 = (float)std::log((double)(float)r0), l1 = (float)std::log((double)(float)r1);
        a.s0 = s0f, a.srange = s1f - s0f, a.lr0 = l0, a.lrange = l1 - l0;
        a.Rh = H_out, a.Rw = W_out;
    } else {
        PCNN_REQUIRE(resize_size >= 1 && resize_size <= RES_MAX_SIDE, PCNN_ERR_ARG, "%s: resize_size = %d: 1 <= resize_size <= %d is required",
                     fn, resize_size, RES_MAX_SIDE);
        const int sh = std::min(H, W), lg = std::max(H, W);
        const long long nl = (long long)((double)((long long)resize_size * lg) / (double)sh);
        PCNN_REQUIRE(nl <= RES_MAX_SIDE, PCNN_ERR_ARG, "%s: resize_size = %d: the longer resized side, %lld, must be <= %d", fn,
                     resize_size, nl, RES_MAX_SIDE);
        a.Rh = W <= H ? (int)nl : resize_size;
        a.Rw = W <= H ? resize_size : (int)nl;
        auto anchor = [](int R, int c) { return c > R ? -((c - R) / 2) : (int)round_half_even((R - c) / 2.0); };
        a.ty = anchor(a.Rh, H_out);
        a.tx = anchor(a.Rw, W_out);
    }
    const int oy = mode == RES_TRAIN ? H_out : a.Rh, ox = mode == RES_TRAIN ? W_out : a.Rw;
    a.taps_y = worst_taps(H, oy);
    a.taps_x = worst_taps(W, ox);
    PCNN_REQUIRE(a.taps_y <= RES_MAX_TAPS && a.taps_x <= RES_MAX_TAPS, PCNN_ERR_ARG,
                 "%s: %d x %d to %d x %d: the whole image needs %d x %d taps, at most %d per axis (2 ceil(in / out) + 1: a downscale of at "
                 "most 16x) is allowed", fn, H, W, oy, ox, a.taps_y, a.taps_x, RES_MAX_TAPS);
    a.n = n;
    a.first = first;
    a.img_bytes = img_bytes;
    a.H = H;
    a.W = W;
    a.C = C;
    a.C_out = C_out;
    a.pitch = (int)pitch;
    a.image_rows = rows;
    a.shuffle = shuffle;
    a.flip = flip;
    a.mode = mode;
    a.H_out = H_out;
    a.W_out = W_out;
    a.b = 0;
    while ((1ULL << (2 * a.b)) < (unsigned long long)n) ++a.b;
    int rpc = std::min(H_out, RES_MAX_RPC);
    while (rpc > 1 && res_smem(a, rpc, rows_cap(H, oy, rpc)) > RES_SMEM) --rpc;
    const long long smem = res_smem(a, rpc, rows_cap(H, oy, rpc));
    PCNN_REQUIRE(smem <= RES_SMEM, PCNN_ERR_ARG,
                 "%s: W_out C = %d x %d: one output row of the whole image needs %lld bytes of shared memory, at most %d are available", fn,
                 W_out, C, smem, RES_SMEM);
    a.rpc = rpc;
    a.rows_cap = rows_cap(H, oy, rpc);
    a.row_blocks = (H_out + rpc - 1) / rpc;
    a.units = (long long)N * a.row_blocks;
    s->vec = row_elems % 8 == 0 ? 8 : 1;
    a.vpr = (int)(row_elems / s->vec);
    s->grid = (int)std::min(AUG_MAX_GRID, a.units);
    s->smem = (int)smem;
    for (int c = 0; c < C; ++c)
        for (int u = 0; u < 256; ++u) a.lut[c * 256 + u] = bf16_rn(aug_value(mean, std_, c, u));
    return PCNN_OK;
}

// the launch after the budget check; the caller holds the device guard
int res_launch(const char *fn, pcnn_ctx *ctx, const ResShape &s) {
    cudaFuncAttributes fa;
    PCNN_CUDA(cudaFuncGetAttributes(&fa, s.vec == 8 ? k_augment_resized<8> : k_augment_resized<1>));
    PCNN_REQUIRE(fa.sharedSizeBytes + (size_t)RES_SMEM <= (size_t)RES_SMEM_LIMIT && s.smem <= fa.maxDynamicSharedSizeBytes, PCNN_ERR_CUDA,
                 "%s: the kernel's %zu bytes of static shared memory leave %d dynamic bytes, below the %d the budget assumes", fn,
                 fa.sharedSizeBytes, fa.maxDynamicSharedSizeBytes, RES_SMEM);
    if (s.vec == 8)
        k_augment_resized<8><<<s.grid, AUG_THREADS, s.smem, ctx->stream>>>(s.a);
    else
        k_augment_resized<1><<<s.grid, AUG_THREADS, s.smem, ctx->stream>>>(s.a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

}  // namespace

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

extern "C" int pcnn_augment_resized_u8_bf16_info(long long n, int H, int W, int C, long long first, int N, int shuffle, int flip,
                                                 int H_out, int W_out, int C_out, int row_pitch, int image_rows, const float *mean_host,
                                                 const float *std_host, int mode, double scale_lo, double scale_hi, double ratio_lo,
                                                 double ratio_hi, int resize_size, long long *out21, uint16_t *lut_out) {
    const char *fn = "pcnn_augment_resized_u8_bf16_info";
    PCNN_REQUIRE(out21, PCNN_ERR_ARG, "%s: NULL out21", fn);
    ResShape s;
    const int rc = res_shape(fn, n, H, W, C, first, N, shuffle, flip, H_out, W_out, C_out, row_pitch, image_rows, mean_host, std_host,
                             mode, scale_lo, scale_hi, ratio_lo, ratio_hi, resize_size, &s);
    if (rc) return rc;
    const ResArgs &a = s.a;
    const long long v[21] = {a.pitch, a.image_rows, a.b, s.vec, s.grid, a.rpc, a.row_blocks, AUG_THREADS, s.smem, a.taps_y, a.taps_x,
                             a.rows_cap, a.Rh, a.Rw, a.ty, a.tx, a.fb_top, a.fb_left, a.fb_h, a.fb_w, RES_SMEM_LIMIT - RES_SMEM};
    memcpy(out21, v, sizeof(v));
    if (lut_out) memcpy(lut_out, a.lut, sizeof(uint16_t) * 256 * C);
    return PCNN_OK;
}

extern "C" int pcnn_augment_resized_u8_bf16(pcnn_ctx *ctx, const uint8_t *images_dev, const uint8_t *labels_dev, long long n, int H, int W,
                                            int C, long long first, int N, int shuffle, int flip, unsigned long long seed,
                                            unsigned long long epoch, const float *mean_host, const float *std_host, void *x_bf16_dev,
                                            int H_out, int W_out, int C_out, int row_pitch, int image_rows, uint8_t *labels_out_dev,
                                            int mode, double scale_lo, double scale_hi, double ratio_lo, double ratio_hi, int resize_size) {
    const char *fn = "pcnn_augment_resized_u8_bf16";
    PCNN_REQUIRE(ctx && images_dev && x_bf16_dev, PCNN_ERR_ARG, "%s: NULL context, images or x (only the labels may be NULL)", fn);
    PCNN_REQUIRE(!labels_dev == !labels_out_dev, PCNN_ERR_ARG, "%s: labels and labels_out must both be NULL or neither", fn);
    ResShape s;
    const int rc = res_shape(fn, n, H, W, C, first, N, shuffle, flip, H_out, W_out, C_out, row_pitch, image_rows, mean_host, std_host,
                             mode, scale_lo, scale_hi, ratio_lo, ratio_hi, resize_size, &s);
    if (rc) return rc;
    PCNN_REQUIRE(aligned16(x_bf16_dev), PCNN_ERR_ARG, "%s: x must be 16-byte aligned", fn);
    ResArgs &a = s.a;
    const size_t xbytes = (((size_t)N - 1) * a.image_rows * a.pitch + (size_t)(H_out - 1) * a.pitch + (size_t)W_out * C_out) * 2;
    PCNN_REQUIRE(disjoint(x_bf16_dev, xbytes, images_dev, (size_t)n * a.img_bytes) && disjoint(x_bf16_dev, xbytes, labels_out_dev, N),
                 PCNN_ERR_ARG, "%s: overlapping buffers: x must share no byte with images or labels_out", fn);
    PCNN_REQUIRE(disjoint(labels_out_dev, N, labels_dev, n) && disjoint(labels_out_dev, N, images_dev, (size_t)n * a.img_bytes),
                 PCNN_ERR_ARG, "%s: overlapping buffers: labels_out must share no byte with labels or images", fn);
    a.img = images_dev;
    a.lab = labels_dev;
    a.x = static_cast<__nv_bfloat16 *>(x_bf16_dev);
    a.lab_out = labels_out_dev;
    a.k0 = (unsigned)seed;
    a.k1 = (unsigned)(seed >> 32);
    a.e0 = (unsigned)epoch;
    a.e1 = (unsigned)(epoch >> 32);
    pcnn_device_guard dg(ctx->device);
    return res_launch(fn, ctx, s);
}

// ------------------------------------------------------------------------------------------------ TrivialAugmentWide, RandomErasing
// pcnn_augment_trivial_u8_bf16: the plain or the resized call's geometry, then torchvision's TrivialAugmentWide on the uint8 crop,
// the table, and RandomErasing(value = 0) on the normalised values.  The geometry runs as k_augment<., MIX_NONE> or
// k_augment_resized with the identity table (bf16 bits u for byte u) into a caller-owned uint16 workspace [N][h][ws_pitch] at
// C_out = C, so its bytes are those kernels' own.  k_trivial then takes one image per CTA: it stages the crop's bytes in shared
// memory, draws the op and the erase box, builds the op's histogram (integer shared atomics: order-free) and byte map, and writes
// each output element from one gather over the staged crop.
namespace {

constexpr int TA_THREADS = 512;
constexpr int TA_OPS = 14, TA_BINS = 31;
constexpr int TA_MAX_PIXELS = 65536;          // h w: the Contrast mean's fp32 sum of bytes stays exact (h w 255 < 2^24)
constexpr int TA_SMEM_LIMIT = 227 * 1024;     // static + dynamic shared memory a CTA may opt into on an H100
constexpr unsigned DOMAIN_TA = 0xC0000000u;   // counter word 1 of trivial block k: DOMAIN_TA | (16 + k) << 24 | i hi, i < 2^56
constexpr int TA_NONE = 0, TA_NEAREST = 1, TA_BILINEAR = 2;
enum TaOp {
    OP_IDENTITY, OP_SHEAR_X, OP_SHEAR_Y, OP_TRANSLATE_X, OP_TRANSLATE_Y, OP_ROTATE, OP_BRIGHTNESS, OP_COLOR, OP_CONTRAST,
    OP_SHARPNESS, OP_POSTERIZE, OP_SOLARIZE, OP_AUTOCONTRAST, OP_EQUALIZE
};

// one (op, bin, sign) of the host table.  Geometric ops: the grid's rescaled inverse matrix, gx = x v0 + y v1 + v2 and
// gy = x v3 + y v4 + v5.  Brightness, Color, Contrast, Sharpness: v0 = RN32(ratio), v1 = RN32(1 - ratio).  Posterize: v0 = the
// mask.  Solarize: v0 = the least byte that is inverted (256: none).
struct TaEntry {
    float v[6];
};

struct TaArgs : AugArgs {                     // AugArgs' permutation, keys and the output's layout and table, H x W the crop
    const unsigned short *ws;                 // [N][H][ws_pitch]: the geometry's bytes
    long long ws_image;                       // H ws_pitch
    int ws_pitch, trivial, erase;
    float erase_p, es0, esr, el0, elr;        // RN32(p), then the erase box's (low, range) pairs as the resized call's
    TaEntry tab[TA_OPS * TA_BINS * 2];        // [op][bin][sign]
};

struct TaShared {
    unsigned short lut[4 * 256];              // the table composed with the op's byte map
    int hist[3][256];
    float fmin[3], fscale[3];
    int step[3];
    unsigned long long i;
    int op, bin, sign, erase, et, el, eh, ew;
    float mean;
};

__device__ __forceinline__ float unit24(unsigned u) { return __fmul_rn((float)(u >> 8), 5.96046448e-08f); }

// _blend on bytes: RN(RN(r a) + RN(s b)), clamped to [0, 255], truncated
__device__ __forceinline__ unsigned blend_u8(float a, float b, float r, float s) {
    return (unsigned)fminf(fmaxf(__fadd_rn(__fmul_rn(r, a), __fmul_rn(s, b)), 0.0f), 255.0f);
}

// rgb_to_grayscale on bytes: RN(RN(RN(0.2989 r) + RN(0.587 g)) + RN(0.114 b)), truncated
__device__ __forceinline__ unsigned gray_u8(const uint8_t *p) {
    return (unsigned)__fadd_rn(__fadd_rn(__fmul_rn(0.2989f, (float)p[0]), __fmul_rn(0.587f, (float)p[1])), __fmul_rn(0.114f, (float)p[2]));
}

// the byte at (y, x, c) of the transformed crop for the gather ops (geometric, Color, Sharpness); the point ops read img as is
__device__ __forceinline__ unsigned ta_byte(const uint8_t *img, const TaArgs &a, const TaEntry &e, int op, int y, int x, int c) {
    const int h = a.H, w = a.W, C = a.C;
    const unsigned u = img[(y * w + x) * C + c];
    if (op >= OP_SHEAR_X && op <= OP_ROTATE) {
        const float bx = __fadd_rn((float)x, 0.5f - 0.5f * (float)w), by = __fadd_rn((float)y, 0.5f - 0.5f * (float)h);
        const float gx = __fadd_rn(__fadd_rn(__fmul_rn(bx, e.v[0]), __fmul_rn(by, e.v[1])), e.v[2]);
        const float gy = __fadd_rn(__fadd_rn(__fmul_rn(bx, e.v[3]), __fmul_rn(by, e.v[4])), e.v[5]);
        const float ix = __fsub_rn(__fmul_rn(__fadd_rn(gx, 1.0f), 0.5f * (float)w), 0.5f);
        const float iy = __fsub_rn(__fmul_rn(__fadd_rn(gy, 1.0f), 0.5f * (float)h), 0.5f);
        auto at = [&](float fy, float fx) -> float {
            return fx >= 0.0f && fx < (float)w && fy >= 0.0f && fy < (float)h ? (float)img[((int)fy * w + (int)fx) * C + c] : 0.0f;
        };
        if (a.trivial == TA_NEAREST) return (unsigned)at(rintf(iy), rintf(ix));
        const float x0 = floorf(ix), y0 = floorf(iy);
        const float tw = __fsub_rn(ix, x0), te = __fsub_rn(1.0f, tw), tn = __fsub_rn(iy, y0), ts = __fsub_rn(1.0f, tn);
        float v = __fmul_rn(at(y0, x0), __fmul_rn(ts, te));
        v = __fadd_rn(v, __fmul_rn(at(y0, x0 + 1.0f), __fmul_rn(ts, tw)));
        v = __fadd_rn(v, __fmul_rn(at(y0 + 1.0f, x0), __fmul_rn(tn, te)));
        v = __fadd_rn(v, __fmul_rn(at(y0 + 1.0f, x0 + 1.0f), __fmul_rn(tn, tw)));
        return (unsigned)fminf(rintf(v), 255.0f);
    }
    if (op == OP_COLOR) return C == 3 ? blend_u8((float)u, (float)gray_u8(img + (y * w + x) * 3), e.v[0], e.v[1]) : u;
    if (op == OP_SHARPNESS) {
        if (h <= 2 || w <= 2) return u;
        unsigned b = u;
        if (y > 0 && y < h - 1 && x > 0 && x < w - 1) {
            const float w1 = 0.0769230798f, w5 = 0.384615391f;     // RN32(1 / 13), RN32(5 / 13): the kernel / its sum
            float acc = 0.0f;
#pragma unroll
            for (int k = 0; k < 9; ++k) {
                const float t = __fmul_rn(k == 4 ? w5 : w1, (float)img[((y + k / 3 - 1) * w + x + k % 3 - 1) * C + c]);
                acc = k == 0 ? t : __fadd_rn(acc, t);
            }
            b = (unsigned)fminf(rintf(acc), 255.0f);
        }
        return blend_u8((float)u, (float)b, e.v[0], e.v[1]);
    }
    return u;
}

template <int VEC>
__global__ void __launch_bounds__(TA_THREADS) k_trivial(const __grid_constant__ TaArgs a) {
    __shared__ TaShared sh;
    extern __shared__ __align__(16) uint8_t img[];                              // [H][W][C]
    const int h = a.H, w = a.W, C = a.C, wC = w * C, hw = h * w;
    for (long long j = blockIdx.x; j < a.units; j += gridDim.x) {
        if (threadIdx.x == 0) {
            const unsigned long long e = (unsigned long long)(a.first + j);
            const unsigned long long i = a.shuffle ? permute(e, a) : e;
            const unsigned lo = (unsigned)i, hi = (unsigned)(i >> 32);
            const uint4 d = philox4x32_10(lo, DOMAIN_TA | 16u << 24 | hi, a.e0, a.e1, a.k0, a.k1);
            sh.op = a.trivial ? (int)__umulhi(d.x, TA_OPS) : OP_IDENTITY;
            sh.bin = (int)__umulhi(d.y, TA_BINS);
            sh.sign = (int)(d.z >> 31);
            int erase = a.erase && unit24(d.w) < a.erase_p, et = 0, el = 0, eh = 0, ew = 0;
            if (erase) {
                erase = 0;
                const double area = __dmul_rn((double)h, (double)w);
                uint4 b = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 1
                for (int t = 0; t < BOX_ATTEMPTS && !erase; ++t) {
                    if ((t & 1) == 0) b = philox4x32_10(lo, DOMAIN_TA | (unsigned)(17 + t / 2) << 24 | hi, a.e0, a.e1, a.k0, a.k1);
                    const float s = __fadd_rn(__fmul_rn(unit24((t & 1) ? b.z : b.x), a.esr), a.es0);
                    const float lr = __fadd_rn(__fmul_rn(unit24((t & 1) ? b.w : b.y), a.elr), a.el0);
                    const double aspect = (double)exp_f32(lr), ea = __dmul_rn(area, (double)s);
                    const double ch = rint(__dsqrt_rn(__dmul_rn(ea, aspect))), cw = rint(__dsqrt_rn(__ddiv_rn(ea, aspect)));
                    if (ch < (double)h && cw < (double)w) {
                        eh = (int)ch;
                        ew = (int)cw;
                        const uint4 r = philox4x32_10(lo, DOMAIN_TA | (unsigned)(17 + BOX_ATTEMPTS / 2) << 24 | hi, a.e0, a.e1, a.k0, a.k1);
                        et = (int)__umulhi(r.x, (unsigned)(h - eh + 1));
                        el = (int)__umulhi(r.y, (unsigned)(w - ew + 1));
                        erase = 1;
                    }
                }
            }
            sh.i = i;
            sh.erase = erase, sh.et = et, sh.el = el, sh.eh = eh, sh.ew = ew;
        }
        for (int t = threadIdx.x; t < 3 * 256; t += TA_THREADS) (&sh.hist[0][0])[t] = 0;
        const unsigned short *ws = a.ws + j * a.ws_image;
        if ((wC & 7) == 0) {
            const int vr = wC >> 3;
            for (int t = threadIdx.x; t < h * vr; t += TA_THREADS) {
                const int r = t / vr, k = (t - r * vr) << 3;
                const uint4 v = *reinterpret_cast<const uint4 *>(ws + (long long)r * a.ws_pitch + k);
                uint2 o;
                o.x = (v.x & 0xFFu) | (v.x >> 8 & 0xFF00u) | (v.y & 0xFFu) << 16 | (v.y >> 16 & 0xFFu) << 24;
                o.y = (v.z & 0xFFu) | (v.z >> 8 & 0xFF00u) | (v.w & 0xFFu) << 16 | (v.w >> 16 & 0xFFu) << 24;
                *reinterpret_cast<uint2 *>(img + r * wC + k) = o;
            }
        } else {
            for (int t = threadIdx.x; t < h * wC; t += TA_THREADS) {
                const int r = t / wC;
                img[t] = (uint8_t)ws[(long long)r * a.ws_pitch + (t - r * wC)];
            }
        }
        __syncthreads();
        const int op = sh.op;
        const TaEntry &e = a.tab[(op * TA_BINS + sh.bin) * 2 + sh.sign];
        if (op == OP_CONTRAST) {
            for (int p = threadIdx.x; p < hw; p += TA_THREADS) atomicAdd(&sh.hist[0][C == 3 ? gray_u8(img + p * 3) : img[p]], 1);
        } else if (op == OP_AUTOCONTRAST || op == OP_EQUALIZE) {
            for (int t = threadIdx.x; t < hw * C; t += TA_THREADS) atomicAdd(&sh.hist[t % C][img[t]], 1);
        }
        __syncthreads();
        if (op == OP_CONTRAST && threadIdx.x == 0) {
            long long sum = 0;
            for (int g = 0; g < 256; ++g) sum += (long long)g * sh.hist[0][g];
            sh.mean = __fdiv_rn((float)sum, (float)hw);                // exact sum: hw 255 < 2^24
        } else if (op == OP_AUTOCONTRAST && threadIdx.x < C) {
            const int *hc = sh.hist[threadIdx.x];
            int lo = 0, hi = 255;
            while (hc[lo] == 0) ++lo;
            while (hc[hi] == 0) --hi;
            sh.fmin[threadIdx.x] = hi == lo ? 0.0f : (float)lo;
            sh.fscale[threadIdx.x] = hi == lo ? 1.0f : __fmul_rn(__frcp_rn((float)(hi - lo)), 255.0f);
        } else if (op == OP_EQUALIZE && threadIdx.x < C) {
            int *hc = sh.hist[threadIdx.x];
            int hi = 255;
            while (hc[hi] == 0) --hi;
            int cum = 0;
            for (int u = 0; u < 256; ++u) cum += hc[u], hc[u] = cum;
            sh.step[threadIdx.x] = (cum - (hc[hi] - (hi ? hc[hi - 1] : 0))) / 255;
        }
        __syncthreads();
        for (int t = threadIdx.x; t < C * 256; t += TA_THREADS) {
            const int c = t >> 8;
            const unsigned u = t & 255;
            unsigned b = u;
            if (op == OP_BRIGHTNESS) b = blend_u8((float)u, 0.0f, e.v[0], e.v[1]);
            else if (op == OP_CONTRAST) b = blend_u8((float)u, sh.mean, e.v[0], e.v[1]);
            else if (op == OP_POSTERIZE) b = u & (unsigned)e.v[0];
            else if (op == OP_SOLARIZE) b = u >= (unsigned)e.v[0] ? 255u - u : u;
            else if (op == OP_AUTOCONTRAST)
                b = (unsigned)fminf(fmaxf(__fmul_rn(__fsub_rn((float)u, sh.fmin[c]), sh.fscale[c]), 0.0f), 255.0f);
            else if (op == OP_EQUALIZE && sh.step[c] != 0)
                b = u == 0 ? 0u : (unsigned)min((sh.hist[c][u - 1] + sh.step[c] / 2) / sh.step[c], 255);
            sh.lut[t] = a.lut[c * 256 + b];
        }
        __syncthreads();
        const bool gather = (op >= OP_SHEAR_X && op <= OP_ROTATE) || op == OP_COLOR || op == OP_SHARPNESS;
        const int erase = sh.erase, et = sh.et, el = sh.el, eb = sh.et + sh.eh, er = sh.el + sh.ew;
        __nv_bfloat16 *xj = a.x + j * a.image_rows * (long long)a.pitch;
        for (int t = threadIdx.x; t < h * a.vpr; t += TA_THREADS) {
            const int r = t / a.vpr;
            const int k = (t - r * a.vpr) * VEC;
            const bool row_erase = erase && r >= et && r < eb;
            int x = k / a.C_out, c = k - x * a.C_out;
            BitsVec<VEC> out;
#pragma unroll
            for (int q = 0; q < VEC; ++q) {
                unsigned short bits = 0;
                if (c < C && !(row_erase && x >= el && x < er))
                    bits = sh.lut[c * 256 + (gather ? ta_byte(img, a, e, op, r, x, c) : img[(r * w + x) * C + c])];
                out.h[q] = bits;
                if (++c == a.C_out) {
                    c = 0;
                    ++x;
                }
            }
            *reinterpret_cast<BitsVec<VEC> *>(xj + (long long)r * a.pitch + k) = out;
        }
        __syncthreads();                                           // the shared state is rewritten by the next image
    }
}

// torch.linspace(0, 0.99, 31) and torch.linspace(0, 32, 31) in fp32, the magnitudes of TrivialAugmentWide._augmentation_space
// (torch's vectorised linspace rounds some bins differently from start + i step; Rotate's and Solarize's bins are exact)
const float TA_MAG_099[TA_BINS] = {
    0.0f, 0.032999999821186066f, 0.06599999964237213f, 0.0989999994635582f, 0.13199999928474426f, 0.16499999165534973f,
    0.1979999989271164f, 0.23100000619888306f, 0.2639999985694885f, 0.296999990940094f, 0.32999998331069946f, 0.3630000054836273f,
    0.3959999978542328f, 0.42899999022483826f, 0.4620000123977661f, 0.4950000047683716f, 0.527999997138977f, 0.5609999895095825f,
    0.593999981880188f, 0.6270000338554382f, 0.6600000262260437f, 0.6930000185966492f, 0.7260000109672546f, 0.7590000033378601f,
    0.7919999957084656f, 0.824999988079071f, 0.8580000400543213f, 0.8910000324249268f, 0.9240000247955322f, 0.9570000171661377f,
    0.9900000095367432f};
const float TA_MAG_32[TA_BINS] = {
    0.0f, 1.0666667222976685f, 2.133333444595337f, 3.200000286102295f, 4.266666889190674f, 5.333333492279053f, 6.40000057220459f,
    7.466667175292969f, 8.533333778381348f, 9.600000381469727f, 10.666666984558105f, 11.733333587646484f, 12.80000114440918f,
    13.866667747497559f, 14.933334350585938f, 15.999999046325684f, 17.066665649414062f, 18.133333206176758f, 19.19999885559082f,
    20.266666412353516f, 21.333332061767578f, 22.399999618530273f, 23.46666717529297f, 24.53333282470703f, 25.600000381469727f,
    26.66666603088379f, 27.733333587646484f, 28.799999237060547f, 29.866666793823242f, 30.933332443237305f, 32.0f};

// the magnitude of (op, bin, sign) as _apply_op receives it: the fp32 bin as a double, negated for a signed op's sign 1
double ta_magnitude(int op, int bin, int sign) {
    double m = 0.0;
    bool signed_op = true;
    switch (op) {
    case OP_SHEAR_X: case OP_SHEAR_Y: case OP_BRIGHTNESS: case OP_COLOR: case OP_CONTRAST: case OP_SHARPNESS: m = TA_MAG_099[bin]; break;
    case OP_TRANSLATE_X: case OP_TRANSLATE_Y: m = TA_MAG_32[bin]; break;
    case OP_ROTATE: m = (double)(4.5f * (float)bin); break;
    case OP_POSTERIZE: m = 8 - (int)std::nearbyint((float)bin / 5.0f), signed_op = false; break;
    case OP_SOLARIZE: m = (double)(255.0f - 8.5f * (float)bin), signed_op = false; break;
    default: signed_op = false;
    }
    return signed_op && sign ? -m : m;
}

// torchvision's _get_inverse_affine_matrix (inverted, scale 1) in double, in its order of operations
void inverse_affine(double cx, double cy, double angle, double tx, double ty, double shear_x, double shear_y, double *m) {
    const double deg2rad = M_PI / 180.0;
    const double rot = angle * deg2rad, sx = shear_x * deg2rad, sy = shear_y * deg2rad;
    const double a = std::cos(rot - sy) / std::cos(sy);
    const double b = -std::cos(rot - sy) * std::tan(sx) / std::cos(sy) - std::sin(rot);
    const double c = std::sin(rot - sy) / std::cos(sy);
    const double d = -std::sin(rot - sy) * std::tan(sx) / std::cos(sy) + std::cos(rot);
    m[0] = d, m[1] = -b, m[2] = 0.0, m[3] = -c, m[4] = a, m[5] = 0.0;
    m[2] += m[0] * (-cx - tx) + m[1] * (-cy - ty);
    m[5] += m[3] * (-cx - tx) + m[4] * (-cy - ty);
    m[2] += cx;
    m[5] += cy;
}

// the entry of (op, bin, sign) for an h x w crop
TaEntry ta_entry(int op, int bin, int sign, int h, int w) {
    TaEntry e{};
    const double mag = ta_magnitude(op, bin, sign);
    if (op >= OP_SHEAR_X && op <= OP_ROTATE) {
        const double rad2deg = 180.0 / M_PI;
        double m[6];
        if (op == OP_SHEAR_X) inverse_affine(-(w * 0.5), -(h * 0.5), 0.0, 0.0, 0.0, std::atan(mag) * rad2deg, 0.0, m);
        else if (op == OP_SHEAR_Y) inverse_affine(-(w * 0.5), -(h * 0.5), 0.0, 0.0, 0.0, 0.0, std::atan(mag) * rad2deg, m);
        else if (op == OP_TRANSLATE_X) inverse_affine(0.0, 0.0, 0.0, (double)(long long)mag, 0.0, 0.0, 0.0, m);
        else if (op == OP_TRANSLATE_Y) inverse_affine(0.0, 0.0, 0.0, 0.0, (double)(long long)mag, 0.0, 0.0, m);
        else inverse_affine(0.0, 0.0, -mag, 0.0, 0.0, 0.0, 0.0, m);
        const float sx = (float)(0.5 * w), sy = (float)(0.5 * h);
        for (int k = 0; k < 3; ++k) e.v[k] = (float)m[k] / sx, e.v[3 + k] = (float)m[3 + k] / sy;
    } else if (op >= OP_BRIGHTNESS && op <= OP_SHARPNESS) {
        const double ratio = 1.0 + mag;
        e.v[0] = (float)ratio;
        e.v[1] = (float)(1.0 - ratio);
    } else if (op == OP_POSTERIZE) {
        e.v[0] = (float)((256 - (1 << (8 - (int)mag))) & 255);
    } else if (op == OP_SOLARIZE) {
        e.v[0] = std::ceil((float)mag);                             // img >= threshold over bytes
    }
    return e;
}

struct TaShape {
    TaArgs a;
    AugShape geo;                     // the plain geometry (resize 0)
    ResShape res;                     // the resized geometry (resize 1)
    int vec, grid, smem;
    long long ws_bytes;
};

// the domain, one message per rule, the geometry's and the output's launches and the table: a function of the arguments alone
int ta_shape(const char *fn, long long n, int H, int W, int C, long long first, int N, int shuffle, int pad, int flip, int resize,
             int H_out, int W_out, double s0, double s1, double r0, double r1, int trivial, double erase_p, double es0, double es1,
             double er0, double er1, int C_out, int row_pitch, int image_rows, const float *mean, const float *std_, TaShape *s) {
    PCNN_REQUIRE(resize == 0 || resize == 1, PCNN_ERR_ARG, "%s: resize = %d: 0 (crop and pad) or 1 (RandomResizedCrop) is required", fn,
                 resize);
    PCNN_REQUIRE(trivial == TA_NONE || trivial == TA_NEAREST || trivial == TA_BILINEAR, PCNN_ERR_ARG,
                 "%s: trivial = %d: 0 (none), 1 (NEAREST) or 2 (BILINEAR) is required", fn, trivial);
    PCNN_REQUIRE(!trivial || C == 1 || C == 3, PCNN_ERR_ARG, "%s: C = %d: TrivialAugmentWide takes C = 1 or 3", fn, C);
    PCNN_REQUIRE(std::isfinite(erase_p) && erase_p >= 0.0 && erase_p <= 1.0, PCNN_ERR_ARG,
                 "%s: erase_p = %g: a finite 0 <= p <= 1 is required", fn, erase_p);
    if (erase_p > 0.0) {
        PCNN_REQUIRE(std::isfinite(es0) && std::isfinite(es1) && es0 >= 0.0 && es0 <= es1 && es1 <= 1.0, PCNN_ERR_ARG,
                     "%s: erase scale = (%g, %g): 0 <= s0 <= s1 <= 1 is required", fn, es0, es1);
        const double lo = 1.1754943508222875e-38, hi = 3.4028234663852886e+38;
        PCNN_REQUIRE(er0 >= lo && er1 <= hi && er0 <= er1, PCNN_ERR_ARG,
                     "%s: erase ratio = (%g, %g): r0 <= r1, each within fp32's normal range [2^-126, 3.4028235e38], is required", fn,
                     er0, er1);
    }
    if (resize) {
        PCNN_REQUIRE(pad == 0, PCNN_ERR_ARG, "%s: pad = %d: a resized batch takes no padding", fn, pad);
        const int rc = res_shape(fn, n, H, W, C, first, N, shuffle, flip, H_out, W_out, C, 0, 0, nullptr, nullptr, RES_TRAIN, s0, s1, r0,
                                 r1, 0, &s->res);
        if (rc) return rc;
    } else {
        const int rc = aug_shape(fn, n, H, W, C, first, N, shuffle, pad, flip, C, 0, 0, nullptr, nullptr, &s->geo);
        if (rc) return rc;
        H_out = H, W_out = W;
    }
    AugArgs &g = resize ? static_cast<AugArgs &>(s->res.a) : s->geo.a;
    for (int c = 0; c < C; ++c)
        for (int u = 0; u < 256; ++u) g.lut[c * 256 + u] = (unsigned short)u;
    AugShape out;
    const int rc = aug_shape(fn, n, H_out, W_out, C, first, N, shuffle, 0, 0, C_out, row_pitch, image_rows, mean, std_, &out);
    if (rc) return rc;
    const long long hw = (long long)H_out * W_out;
    PCNN_REQUIRE(hw <= TA_MAX_PIXELS, PCNN_ERR_ARG, "%s: the crop is %d x %d: at most %d pixels (256 x 256) are allowed", fn, H_out, W_out,
                 TA_MAX_PIXELS);
    const long long smem = (hw * C + 15) / 16 * 16, smem_max = TA_SMEM_LIMIT - (long long)((sizeof(TaShared) + 15) / 16 * 16);
    PCNN_REQUIRE(smem <= smem_max, PCNN_ERR_ARG,
                 "%s: the crop is %d x %d x %d: its %lld bytes, staged in shared memory, must be <= %lld (227 KB less the kernel's "
                 "static shared memory)", fn, H_out, W_out, C, smem, smem_max);
    TaArgs &a = s->a;
    memset(&a, 0, sizeof(a));
    static_cast<AugArgs &>(a) = out.a;
    a.units = N;                                              // one image per CTA
    a.ws_pitch = g.pitch;
    a.ws_image = (long long)H_out * g.pitch;
    a.trivial = trivial;
    a.erase = erase_p > 0.0;
    a.erase_p = (float)erase_p;
    if (a.erase) {
        const float s0f = (float)es0, s1f = (float)es1, l0 = (float)std::log((double)(float)er0), l1 = (float)std::log((double)(float)er1);
        a.es0 = s0f, a.esr = s1f - s0f, a.el0 = l0, a.elr = l1 - l0;
    }
    for (int op = 0; op < TA_OPS; ++op)
        for (int bin = 0; bin < TA_BINS; ++bin)
            for (int sign = 0; sign < 2; ++sign) a.tab[(op * TA_BINS + bin) * 2 + sign] = ta_entry(op, bin, sign, H_out, W_out);
    s->vec = out.vec;
    s->grid = (int)std::min<long long>(AUG_MAX_GRID, N);
    s->smem = (int)smem;
    s->ws_bytes = (long long)N * a.ws_image * 2;
    return PCNN_OK;
}

}  // namespace

extern "C" int pcnn_augment_trivial_u8_bf16_info(long long n, int H, int W, int C, long long first, int N, int shuffle, int pad, int flip,
                                                 int resize, int H_out, int W_out, double scale_lo, double scale_hi, double ratio_lo,
                                                 double ratio_hi, int trivial, double erase_p, double erase_scale_lo,
                                                 double erase_scale_hi, double erase_ratio_lo, double erase_ratio_hi, int C_out,
                                                 int row_pitch, int image_rows, const float *mean_host, const float *std_host,
                                                 long long *out12, float *table_out, uint16_t *lut_out) {
    const char *fn = "pcnn_augment_trivial_u8_bf16_info";
    PCNN_REQUIRE(out12, PCNN_ERR_ARG, "%s: NULL out12", fn);
    const std::unique_ptr<TaShape> s(new TaShape);             // the table makes it 26 KB
    const int rc = ta_shape(fn, n, H, W, C, first, N, shuffle, pad, flip, resize, H_out, W_out, scale_lo, scale_hi, ratio_lo, ratio_hi,
                            trivial, erase_p, erase_scale_lo, erase_scale_hi, erase_ratio_lo, erase_ratio_hi, C_out, row_pitch,
                            image_rows, mean_host, std_host, s.get());
    if (rc) return rc;
    const TaArgs &a = s->a;
    const long long v[12] = {a.pitch, a.image_rows, a.H, a.W, a.ws_pitch, s->ws_bytes, s->vec, s->grid, TA_THREADS, s->smem,
                             (long long)((sizeof(TaShared) + 15) / 16 * 16), (long long)sizeof(TaArgs)};
    memcpy(out12, v, sizeof(v));
    if (table_out) memcpy(table_out, a.tab, sizeof(a.tab));
    if (lut_out) memcpy(lut_out, a.lut, sizeof(uint16_t) * 256 * C);
    return PCNN_OK;
}

extern "C" int pcnn_augment_trivial_u8_bf16(pcnn_ctx *ctx, const uint8_t *images_dev, const uint8_t *labels_dev, long long n, int H, int W,
                                            int C, long long first, int N, int shuffle, int pad, int flip, unsigned long long seed,
                                            unsigned long long epoch, const float *mean_host, const float *std_host, void *x_bf16_dev,
                                            int C_out, int row_pitch, int image_rows, uint8_t *labels_out_dev, int resize, int H_out,
                                            int W_out, double scale_lo, double scale_hi, double ratio_lo, double ratio_hi, int trivial,
                                            double erase_p, double erase_scale_lo, double erase_scale_hi, double erase_ratio_lo,
                                            double erase_ratio_hi, void *workspace_dev, long long workspace_bytes) {
    const char *fn = "pcnn_augment_trivial_u8_bf16";
    PCNN_REQUIRE(ctx && images_dev && x_bf16_dev && workspace_dev, PCNN_ERR_ARG,
                 "%s: NULL context, images, x or workspace (only the labels may be NULL)", fn);
    PCNN_REQUIRE(!labels_dev == !labels_out_dev, PCNN_ERR_ARG, "%s: labels and labels_out must both be NULL or neither", fn);
    const std::unique_ptr<TaShape> holder(new TaShape);
    TaShape &s = *holder;
    const int rc = ta_shape(fn, n, H, W, C, first, N, shuffle, pad, flip, resize, H_out, W_out, scale_lo, scale_hi, ratio_lo, ratio_hi,
                            trivial, erase_p, erase_scale_lo, erase_scale_hi, erase_ratio_lo, erase_ratio_hi, C_out, row_pitch,
                            image_rows, mean_host, std_host, &s);
    if (rc) return rc;
    TaArgs &a = s.a;
    PCNN_REQUIRE(aligned16(x_bf16_dev) && aligned16(workspace_dev), PCNN_ERR_ARG, "%s: x and the workspace must be 16-byte aligned", fn);
    PCNN_REQUIRE(workspace_bytes >= s.ws_bytes, PCNN_ERR_ARG, "%s: workspace_bytes = %lld: at least %lld (N h ws_pitch 2) are required", fn,
                 workspace_bytes, s.ws_bytes);
    const size_t xbytes = (((size_t)N - 1) * a.image_rows * a.pitch + (size_t)(a.H - 1) * a.pitch + (size_t)a.W * a.C_out) * 2;
    const size_t ibytes = (size_t)n * H * W * C, wbytes = (size_t)s.ws_bytes;
    PCNN_REQUIRE(disjoint(x_bf16_dev, xbytes, images_dev, ibytes) && disjoint(x_bf16_dev, xbytes, labels_out_dev, N) &&
                     disjoint(x_bf16_dev, xbytes, workspace_dev, wbytes),
                 PCNN_ERR_ARG, "%s: overlapping buffers: x must share no byte with images, labels_out or the workspace", fn);
    PCNN_REQUIRE(disjoint(labels_out_dev, N, labels_dev, n) && disjoint(labels_out_dev, N, images_dev, ibytes) &&
                     disjoint(labels_out_dev, N, workspace_dev, wbytes),
                 PCNN_ERR_ARG, "%s: overlapping buffers: labels_out must share no byte with labels, images or the workspace", fn);
    PCNN_REQUIRE(disjoint(workspace_dev, wbytes, images_dev, ibytes) && disjoint(workspace_dev, wbytes, labels_dev, n), PCNN_ERR_ARG,
                 "%s: overlapping buffers: the workspace must share no byte with images or labels", fn);
    AugArgs &g = resize ? static_cast<AugArgs &>(s.res.a) : s.geo.a;
    g.img = images_dev;
    g.lab = labels_dev;
    g.x = static_cast<__nv_bfloat16 *>(workspace_dev);
    g.lab_out = labels_out_dev;
    a.ws = static_cast<const unsigned short *>(workspace_dev);
    a.x = static_cast<__nv_bfloat16 *>(x_bf16_dev);
    g.k0 = a.k0 = (unsigned)seed;
    g.k1 = a.k1 = (unsigned)(seed >> 32);
    g.e0 = a.e0 = (unsigned)epoch;
    g.e1 = a.e1 = (unsigned)(epoch >> 32);
    pcnn_device_guard dg(ctx->device);
    auto kern = s.vec == 8 ? k_trivial<8> : k_trivial<1>;
    cudaFuncAttributes fa;
    PCNN_CUDA(cudaFuncGetAttributes(&fa, kern));
    PCNN_REQUIRE(fa.sharedSizeBytes <= sizeof(TaShared) + 15, PCNN_ERR_CUDA,
                 "%s: the kernel's %zu bytes of static shared memory exceed the %zu the budget assumes", fn, fa.sharedSizeBytes,
                 sizeof(TaShared));
    PCNN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, s.smem));
    const int grc = resize ? res_launch(fn, ctx, s.res) : aug_launch(ctx, s.geo);   // only after every check has passed
    if (grc) return grc;
    kern<<<s.grid, TA_THREADS, s.smem, ctx->stream>>>(a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
