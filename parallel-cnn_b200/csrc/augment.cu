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
    cudaFuncAttributes fa;
    PCNN_CUDA(cudaFuncGetAttributes(&fa, s.vec == 8 ? k_augment_resized<8> : k_augment_resized<1>));
    PCNN_REQUIRE(fa.sharedSizeBytes + (size_t)RES_SMEM <= (size_t)RES_SMEM_LIMIT && s.smem <= fa.maxDynamicSharedSizeBytes, PCNN_ERR_CUDA,
                 "%s: the kernel's %zu bytes of static shared memory leave %d dynamic bytes, below the %d the budget assumes", fn,
                 fa.sharedSizeBytes, fa.maxDynamicSharedSizeBytes, RES_SMEM);
    if (s.vec == 8)
        k_augment_resized<8><<<s.grid, AUG_THREADS, s.smem, ctx->stream>>>(a);
    else
        k_augment_resized<1><<<s.grid, AUG_THREADS, s.smem, ctx->stream>>>(a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
