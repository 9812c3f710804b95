// parallel-cnn_b200/csrc/pool_nhwc.cu -- max pooling between bf16 NHWC convolution layers (pcnn_maxpool_nhwc_bf16_fwd / _bwd):
// x is what the forwards write as y, the pooled y is what a plan reads as x, and dx is what the layer gradients read as dy, so a
// pool sits between two ConvLayers with no copies.  The contract is in include/pcnn.h.
//
// Both passes are HBM-bound.  With C % 8 == 0 a thread moves 16-byte vectors of 8 channels of one pixel, otherwise single
// elements.  Forward: one thread per (output pixel, channel group) scans its window in (r, s) order and stores y once and the
// argmax bytes once.  Backward: a gather, one thread per (input pixel, channel group): it visits the windows that contain its
// pixel in ascending (p, q), adds the dy of those whose argmax points at it in fp32 and writes dx once, so every element of
// dx is written (0 where nothing points), with no memset and no atomics.  The work of a thread depends only on the shape: the
// bits are the same on every run and every H100.
//
// Average pooling (pcnn_avgpool_nhwc_bf16_fwd / _bwd) is the same two passes with a sum in place of the compare and no argmax.
// Global average pooling (pcnn_global_avgpool_nhwc_bf16_fwd / _bwd) writes y in the x layout of a LinearLayer with P = Q = 1:
// its forward is a reduction over the pixels of an image (partition at k_gap_fwd), its backward a broadcast.
#include "pcnn_internal.h"

#include <cuda_bf16.h>

#include <algorithm>

namespace {

constexpr int POOL_THREADS = 256;
constexpr int POOL_MAX_TAPS = 7;

template <int VEC>
struct alignas(2 * VEC) BfVec {
    __nv_bfloat16 h[VEC];
};
template <int VEC>
struct alignas(VEC) ByteVec {
    uint8_t b[VEC];
};

struct PoolArgs {
    int H, W, C, R, S, stride, pad_h, pad_w, P, Q;
    int G;                  // channel groups of VEC channels
    int pitch, rows;        // pitched layout of y / dy
    int work;               // threads one image needs: P * Q * G (forward) or H * W * G (backward)
    int blocks;             // CTAs per image
};

template <int VEC>
__global__ void __launch_bounds__(POOL_THREADS) k_maxpool_nhwc_fwd(const __nv_bfloat16 *__restrict__ x, __nv_bfloat16 *__restrict__ y,
                                                                   uint8_t *__restrict__ argmax, PoolArgs a) {
    const int n = blockIdx.x / a.blocks;
    const int i = (blockIdx.x - n * a.blocks) * POOL_THREADS + threadIdx.x;
    if (i >= a.work) return;
    const int g = i % a.G, pq = i / a.G, q = pq % a.Q, p = pq / a.Q;
    const int h0 = p * a.stride - a.pad_h, w0 = q * a.stride - a.pad_w;
    const int r0 = max(0, -h0), r1 = min(a.R, a.H - h0), s0 = max(0, -w0), s1 = min(a.S, a.W - w0);
    const __nv_bfloat16 *xi = x + (long)n * a.H * a.W * a.C + g * VEC;
    float m[VEC];
    BfVec<VEC> best;
    ByteVec<VEC> arg;
#pragma unroll
    for (int c = 0; c < VEC; ++c) {
        m[c] = -INFINITY;
        best.h[c] = __ushort_as_bfloat16(0xFF80);          // -Inf: the first in-image element of an all -Inf window
        arg.b[c] = (uint8_t)(r0 * a.S + s0);
    }
    for (int r = r0; r < r1; ++r) {
        const __nv_bfloat16 *row = xi + (long)(h0 + r) * a.W * a.C;
        for (int s = s0; s < s1; ++s) {
            const BfVec<VEC> v = *reinterpret_cast<const BfVec<VEC> *>(row + (long)(w0 + s) * a.C);
#pragma unroll
            for (int c = 0; c < VEC; ++c) {
                const float f = __bfloat162float(v.h[c]);
                if (f > m[c] || f != f) {                  // first maximum wins a tie; the last NaN wins
                    m[c] = f;
                    best.h[c] = v.h[c];
                    arg.b[c] = (uint8_t)(r * a.S + s);
                }
            }
        }
    }
    *reinterpret_cast<BfVec<VEC> *>(y + (long)n * a.rows * a.pitch + (long)p * a.pitch + q * a.C + g * VEC) = best;
    if (argmax) *reinterpret_cast<ByteVec<VEC> *>(argmax + (((long)n * a.P + p) * a.Q + q) * a.C + g * VEC) = arg;
}

template <int VEC>
__global__ void __launch_bounds__(POOL_THREADS) k_maxpool_nhwc_bwd(const __nv_bfloat16 *__restrict__ dy, const uint8_t *__restrict__ argmax,
                                                                   __nv_bfloat16 *__restrict__ dx, PoolArgs a) {
    const int n = blockIdx.x / a.blocks;
    const int i = (blockIdx.x - n * a.blocks) * POOL_THREADS + threadIdx.x;
    if (i >= a.work) return;
    const int g = i % a.G, hw = i / a.G, w = hw % a.W, h = hw / a.W;
    // windows p with p * stride - pad_h <= h <= p * stride - pad_h + R - 1, inside [0, P)
    const int nh = h + a.pad_h - a.R + 1, nw = w + a.pad_w - a.S + 1;
    const int p0 = nh <= 0 ? 0 : (nh + a.stride - 1) / a.stride, p1 = min(a.P - 1, (h + a.pad_h) / a.stride);
    const int q0 = nw <= 0 ? 0 : (nw + a.stride - 1) / a.stride, q1 = min(a.Q - 1, (w + a.pad_w) / a.stride);
    const uint8_t *am = argmax + (long)n * a.P * a.Q * a.C + g * VEC;
    const __nv_bfloat16 *dyi = dy + (long)n * a.rows * a.pitch + g * VEC;
    float acc[VEC];
    BfVec<VEC> first;
    unsigned hit = 0, multi = 0;                           // channels with >= 1 / >= 2 terms
#pragma unroll
    for (int c = 0; c < VEC; ++c) {
        acc[c] = 0.0f;
        first.h[c] = __ushort_as_bfloat16(0);
    }
    for (int p = p0; p <= p1; ++p) {
        const int r = h + a.pad_h - p * a.stride;
        for (int q = q0; q <= q1; ++q) {
            const int t = r * a.S + (w + a.pad_w - q * a.stride);
            // both loads issued together: a dy load that waited for the argmax would serialise two memory latencies
            const ByteVec<VEC> av = *reinterpret_cast<const ByteVec<VEC> *>(am + ((long)p * a.Q + q) * a.C);
            const BfVec<VEC> d = *reinterpret_cast<const BfVec<VEC> *>(dyi + (long)p * a.pitch + q * a.C);
            unsigned match = 0;
#pragma unroll
            for (int c = 0; c < VEC; ++c) match |= (av.b[c] == t ? 1u : 0u) << c;
#pragma unroll
            for (int c = 0; c < VEC; ++c) {
                if (!((match >> c) & 1)) continue;
                const float f = __bfloat162float(d.h[c]);
                if ((hit >> c) & 1) {
                    acc[c] = __fadd_rn(acc[c], f);
                    multi |= 1u << c;
                } else {
                    acc[c] = f;                            // the sum starts from the first term
                    first.h[c] = d.h[c];
                }
            }
            hit |= match;
        }
    }
    BfVec<VEC> out;
#pragma unroll
    for (int c = 0; c < VEC; ++c)
        out.h[c] = ((multi >> c) & 1) ? __float2bfloat16_rn(acc[c]) : ((hit >> c) & 1) ? first.h[c] : __ushort_as_bfloat16(0);
    *reinterpret_cast<BfVec<VEC> *>(dx + (((long)n * a.H + h) * a.W + w) * a.C + g * VEC) = out;
}

// RN(1 / k) for the window counts k = 1..49 (constant-folded in IEEE double)
struct RcpTable {
    double v[POOL_MAX_TAPS * POOL_MAX_TAPS + 1];
};
constexpr RcpTable make_rcp() {
    RcpTable t{};
    for (int k = 1; k <= POOL_MAX_TAPS * POOL_MAX_TAPS; ++k) t.v[k] = 1.0 / k;
    return t;
}
__constant__ RcpTable k_rcp = make_rcp();

// y = bf16_rn(s / cnt): s sums the window's in-image elements in (r, s) order starting from the first, cnt = R S with
// count_include_pad, else the in-image positions (>= 1: pad <= R/2 puts an image element in every window)
template <int VEC>
__global__ void __launch_bounds__(POOL_THREADS) k_avgpool_nhwc_fwd(const __nv_bfloat16 *__restrict__ x, __nv_bfloat16 *__restrict__ y, PoolArgs a,
                                                                   int include_pad) {
    const int n = blockIdx.x / a.blocks;
    const int i = (blockIdx.x - n * a.blocks) * POOL_THREADS + threadIdx.x;
    if (i >= a.work) return;
    const int g = i % a.G, pq = i / a.G, q = pq % a.Q, p = pq / a.Q;
    const int h0 = p * a.stride - a.pad_h, w0 = q * a.stride - a.pad_w;
    const int r0 = max(0, -h0), r1 = min(a.R, a.H - h0), s0 = max(0, -w0), s1 = min(a.S, a.W - w0);
    const int cnt = include_pad ? a.R * a.S : (r1 - r0) * (s1 - s0);
    const __nv_bfloat16 *xi = x + (long)n * a.H * a.W * a.C + g * VEC;
    float acc[VEC];                                        // -0 + f == f for every f: the sum starts from the first term
#pragma unroll
    for (int c = 0; c < VEC; ++c) acc[c] = -0.0f;
    for (int r = r0; r < r1; ++r) {
        const __nv_bfloat16 *row = xi + (long)(h0 + r) * a.W * a.C;
        for (int s = s0; s < s1; ++s) {
            const BfVec<VEC> v = *reinterpret_cast<const BfVec<VEC> *>(row + (long)(w0 + s) * a.C);
#pragma unroll
            for (int c = 0; c < VEC; ++c) acc[c] = __fadd_rn(acc[c], __bfloat162float(v.h[c]));
        }
    }
    BfVec<VEC> out;
#pragma unroll
    for (int c = 0; c < VEC; ++c) out.h[c] = __float2bfloat16_rn(div_rn(acc[c], (double)cnt, k_rcp.v[cnt]));
    *reinterpret_cast<BfVec<VEC> *>(y + (long)n * a.rows * a.pitch + (long)p * a.pitch + q * a.C + g * VEC) = out;
}

// the gather of the forward: dx sums float(dy) / cnt over the windows that contain the pixel in ascending (p, q), each quotient
// rounded, from the first term, rounded to bf16 once; +0 with no term
template <int VEC>
__global__ void __launch_bounds__(POOL_THREADS) k_avgpool_nhwc_bwd(const __nv_bfloat16 *__restrict__ dy, __nv_bfloat16 *__restrict__ dx, PoolArgs a,
                                                                   int include_pad) {
    const int n = blockIdx.x / a.blocks;
    const int i = (blockIdx.x - n * a.blocks) * POOL_THREADS + threadIdx.x;
    if (i >= a.work) return;
    const int g = i % a.G, hw = i / a.G, w = hw % a.W, h = hw / a.W;
    const int nh = h + a.pad_h - a.R + 1, nw = w + a.pad_w - a.S + 1;
    const int p0 = nh <= 0 ? 0 : (nh + a.stride - 1) / a.stride, p1 = min(a.P - 1, (h + a.pad_h) / a.stride);
    const int q0 = nw <= 0 ? 0 : (nw + a.stride - 1) / a.stride, q1 = min(a.Q - 1, (w + a.pad_w) / a.stride);
    const __nv_bfloat16 *dyi = dy + (long)n * a.rows * a.pitch + g * VEC;
    float acc[VEC];                                        // -0 + t == t for every t: the sum starts from the first term
#pragma unroll
    for (int c = 0; c < VEC; ++c) acc[c] = -0.0f;
    for (int p = p0; p <= p1; ++p) {
        const int hs = p * a.stride - a.pad_h;
        const int rows = include_pad ? a.R : min(a.R, a.H - hs) - max(0, -hs);
        for (int q = q0; q <= q1; ++q) {
            const int ws = q * a.stride - a.pad_w;
            const int cnt = include_pad ? a.R * a.S : rows * (min(a.S, a.W - ws) - max(0, -ws));
            const double b = cnt, rb = k_rcp.v[cnt];
            const BfVec<VEC> d = *reinterpret_cast<const BfVec<VEC> *>(dyi + (long)p * a.pitch + q * a.C);
#pragma unroll
            for (int c = 0; c < VEC; ++c) acc[c] = __fadd_rn(acc[c], div_rn(__bfloat162float(d.h[c]), b, rb));
        }
    }
    const bool none = p0 > p1 || q0 > q1;
    BfVec<VEC> out;
#pragma unroll
    for (int c = 0; c < VEC; ++c) out.h[c] = none ? __ushort_as_bfloat16(0) : __float2bfloat16_rn(acc[c]);
    *reinterpret_cast<BfVec<VEC> *>(dx + (((long)n * a.H + h) * a.W + w) * a.C + g * VEC) = out;
}

// Global average pooling.  CTA (n, range, slice) owns the pixels [range * per_cta, (range + 1) * per_cta) of image n and the
// channel groups [slice * Gc, (slice + 1) * Gc); thread t keeps group t % Gc of the pixels lane, lane + lanes, ... (lane = t / Gc,
// lanes = 256 / Gc, GAP_ITERS pixels each), summed from the first; the lanes that hold a pixel are then added in lane order
// through shared memory.  One range per image writes y; more write fp32 slots [n][range][C] that k_gap_finish adds in range order.
// GapArgs, GAP_ITERS and gap_shape are in pcnn_internal.h: the squeeze-and-excitation gate gradient sums in the same partition.
constexpr int GAP_MAX_GROUPS = POOL_THREADS;               // channel groups per CTA: C up to 2048 in one slice on the 16-byte path
static_assert(GAP_THREADS == POOL_THREADS, "the partition of gap_shape is that of a POOL_THREADS CTA");

template <int VEC>
__global__ void __launch_bounds__(POOL_THREADS) k_gap_fwd(const __nv_bfloat16 *__restrict__ x, __nv_bfloat16 *__restrict__ y,
                                                          float *__restrict__ slots, GapArgs a) {
    __shared__ float part[POOL_THREADS * 8];               // [lanes][Gc * VEC]: lanes * Gc <= 256
    constexpr int U = VEC == 8 ? 4 : 8;                    // pixels loaded before any is added
    const int slice = blockIdx.x % a.slices, nr = blockIdx.x / a.slices, rg = nr % a.ranges, n = nr / a.ranges;
    const int lane = threadIdx.x / a.Gc, gl = threadIdx.x % a.Gc, g = slice * a.Gc + gl;
    const int width = a.Gc * VEC, p0 = rg * a.per_cta;
    if (lane < a.lanes && g < a.G && p0 + lane < a.HW) {
        const __nv_bfloat16 *xi = x + (long)n * a.HW * a.C + g * VEC;
        float acc[VEC];
        for (int j0 = 0; j0 < GAP_ITERS; j0 += U) {
            BfVec<VEC> v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int px = min(p0 + lane + (j0 + u) * a.lanes, a.HW - 1);     // past the image: a pixel loaded and not added
                v[u] = *reinterpret_cast<const BfVec<VEC> *>(xi + (long)px * a.C);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (p0 + lane + (j0 + u) * a.lanes >= a.HW) continue;
#pragma unroll
                for (int c = 0; c < VEC; ++c) {
                    const float f = __bfloat162float(v[u].h[c]);
                    acc[c] = j0 + u == 0 ? f : __fadd_rn(acc[c], f);
                }
            }
        }
#pragma unroll
        for (int c = 0; c < VEC; ++c) part[lane * width + gl * VEC + c] = acc[c];
    }
    __syncthreads();
    const int active = min(a.lanes, a.HW - p0);            // lanes holding at least one pixel
    for (int t = threadIdx.x; t < width; t += POOL_THREADS) {
        const int c = slice * width + t;
        if (c >= a.C) break;
        float s = part[t];
        for (int l = 1; l < active; ++l) s = __fadd_rn(s, part[l * width + t]);
        if (a.ranges == 1)
            y[(long)n * a.pitch + c] = __float2bfloat16_rn(div_rn(s, a.hw, a.rhw));
        else
            slots[(long)nr * a.C + c] = s;
    }
}

// one thread per (n, c): the slots of image n added in range order, then y = bf16_rn(s / float(H W))
__global__ void __launch_bounds__(POOL_THREADS) k_gap_finish(const float *__restrict__ slots, __nv_bfloat16 *__restrict__ y, int N, GapArgs a) {
    const long i = (long)blockIdx.x * POOL_THREADS + threadIdx.x;
    if (i >= (long)N * a.C) return;
    const int n = (int)(i / a.C), c = (int)(i - (long)n * a.C);
    const float *sl = slots + (long)n * a.ranges * a.C + c;
    float s = sl[0];
    for (int r = 1; r < a.ranges; ++r) s = __fadd_rn(s, sl[(long)r * a.C]);
    y[(long)n * a.pitch + c] = __float2bfloat16_rn(div_rn(s, a.hw, a.rhw));
}

// dx[n][pixel][c] = bf16_rn(float(dy[n][c]) / float(H W)): one 16-byte store per (pixel, channel group)
template <int VEC>
__global__ void __launch_bounds__(POOL_THREADS) k_gap_bwd(const __nv_bfloat16 *__restrict__ dy, __nv_bfloat16 *__restrict__ dx, GapArgs a,
                                                          int blocks) {
    const int n = blockIdx.x / blocks;
    const int i = (blockIdx.x - n * blocks) * POOL_THREADS + threadIdx.x;
    if (i >= a.HW * a.G) return;
    const int g = i % a.G, px = i / a.G;
    const BfVec<VEC> d = *reinterpret_cast<const BfVec<VEC> *>(dy + (long)n * a.pitch + g * VEC);
    BfVec<VEC> out;
#pragma unroll
    for (int c = 0; c < VEC; ++c) out.h[c] = __float2bfloat16_rn(div_rn(__bfloat162float(d.h[c]), a.hw, a.rhw));
    *reinterpret_cast<BfVec<VEC> *>(dx + ((long)n * a.HW + px) * a.C + g * VEC) = out;
}

struct PoolShape {
    PoolArgs args;
    int vec, cover;         // channels per thread; most windows over one input pixel
};

// windows over one input row (or column) at most: the count is periodic in h with period `stride` away from the edges, so the
// first and the last R + 2 * stride rows hold every value it takes
int max_cover(int H, int R, int stride, int pad, int P) {
    int best = 0;
    auto count = [&](int h) {
        const int nh = h + pad - R + 1;
        const int p0 = nh <= 0 ? 0 : (nh + stride - 1) / stride, p1 = std::min(P - 1, (h + pad) / stride);
        best = std::max(best, p1 - p0 + 1);
    };
    const int span = R + 2 * stride;
    for (int h = 0; h < std::min(H, span); ++h) count(h);
    for (int h = std::max(span, H - span); h < H; ++h) count(h);
    return best;
}

// the domain of pcnn.h, refused with PCNN_ERR_ARG and a message naming `fn`
int pool_shape(const char *fn, int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int row_pitch, int image_rows,
               PoolShape *out) {
    PCNN_REQUIRE(N >= 1 && H >= 1 && W >= 1 && C >= 1, PCNN_ERR_ARG, "%s: N = %d, H = %d, W = %d, C = %d: each must be >= 1", fn, N, H, W,
                 C);
    PCNN_REQUIRE(R >= 1 && R <= POOL_MAX_TAPS && S >= 1 && S <= POOL_MAX_TAPS, PCNN_ERR_ARG,
                 "%s: %dx%d window: 1 <= R, S <= 7 is required", fn, R, S);
    PCNN_REQUIRE(stride >= 1 && stride <= POOL_MAX_TAPS, PCNN_ERR_ARG, "%s: stride %d: 1 <= stride <= 7 is required", fn, stride);
    PCNN_REQUIRE(pad_h >= 0 && pad_h <= R / 2 && pad_w >= 0 && pad_w <= S / 2, PCNN_ERR_ARG,
                 "%s: padding (%d, %d) for a %dx%d window: 0 <= pad_h <= R/2 and 0 <= pad_w <= S/2 are required", fn, pad_h, pad_w, R, S);
    PCNN_REQUIRE(H + 2 * pad_h >= R && W + 2 * pad_w >= S, PCNN_ERR_ARG,
                 "%s: a %dx%d window does not fit the %dx%d image padded by (%d, %d): H + 2 pad_h >= R and W + 2 pad_w >= S are required",
                 fn, R, S, H, W, pad_h, pad_w);
    const int P = (H + 2 * pad_h - R) / stride + 1, Q = (W + 2 * pad_w - S) / stride + 1;
    const int vec = C % 8 == 0 ? 8 : 1, G = C / vec;
    PCNN_REQUIRE((long)H * W * G <= INT32_MAX - POOL_THREADS && (long)P * Q * G <= INT32_MAX - POOL_THREADS && (long)Q * C <= INT32_MAX - 8,
                 PCNN_ERR_ARG,
                 "%s: one %dx%dx%d image exceeds the 32-bit index range of a pass", fn, H, W, C);
    const int qc = Q * C;
    if (row_pitch == 0) row_pitch = (qc + 7) / 8 * 8;
    PCNN_REQUIRE(row_pitch >= qc && row_pitch % 8 == 0, PCNN_ERR_ARG,
                 "%s: row_pitch %d: 0 (Q*C rounded up to 8) or a multiple of 8 that is >= Q*C = %d is required", fn, row_pitch, qc);
    if (image_rows == 0) image_rows = P;
    PCNN_REQUIRE(image_rows >= P, PCNN_ERR_ARG, "%s: image_rows %d: 0 (P) or >= P = %d is required", fn, image_rows, P);
    PoolArgs a{H, W, C, R, S, stride, pad_h, pad_w, P, Q, G, row_pitch, image_rows, 0, 0};
    out->args = a;
    out->vec = vec;
    out->cover = max_cover(H, R, stride, pad_h, P) * max_cover(W, S, stride, pad_w, Q);
    return PCNN_OK;
}

bool overlap(const void *a, size_t na, const void *b, size_t nb) {
    if (!a || !b) return false;
    const uintptr_t pa = (uintptr_t)a, pb = (uintptr_t)b;
    return pa < pb + nb && pb < pa + na;
}

bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// one CTA range per image; the grid is N * blocks CTAs
int pool_grid(const char *fn, int N, PoolArgs *a, int work, unsigned *grid) {
    a->work = work;
    a->blocks = (work + POOL_THREADS - 1) / POOL_THREADS;
    PCNN_REQUIRE((long)N * a->blocks <= INT32_MAX, PCNN_ERR_ARG, "%s: %d images of %d threads exceed the grid", fn, N, work);
    *grid = (unsigned)((long)N * a->blocks);
    return PCNN_OK;
}

// out5 of pcnn_maxpool_nhwc_info and pcnn_avgpool_nhwc_info
int pool_info(const char *fn, int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int row_pitch, int image_rows,
              int *out5) {
    PCNN_REQUIRE(out5, PCNN_ERR_ARG, "%s: NULL out5", fn);
    PoolShape sh;
    int rc = pool_shape(fn, N, H, W, C, R, S, stride, pad_h, pad_w, row_pitch, image_rows, &sh);
    if (rc) return rc;
    out5[0] = sh.args.P;
    out5[1] = sh.args.Q;
    out5[2] = sh.args.pitch;
    out5[3] = sh.vec;
    out5[4] = sh.cover;
    return PCNN_OK;
}

int include_pad_flag(const char *fn, int count_include_pad) {
    PCNN_REQUIRE(count_include_pad == 0 || count_include_pad == 1, PCNN_ERR_ARG, "%s: count_include_pad = %d: 0 or 1 is required", fn,
                 count_include_pad);
    return PCNN_OK;
}

}  // namespace

// the global pool's domain and partition, a function of (N, H, W, C) and the row pitch alone (pcnn_internal.h)
int gap_shape(const char *fn, int N, int H, int W, int C, int row_pitch, GapArgs *a) {
    PCNN_REQUIRE(N >= 1 && H >= 1 && W >= 1 && C >= 1, PCNN_ERR_ARG, "%s: N = %d, H = %d, W = %d, C = %d: each must be >= 1", fn, N, H, W,
                 C);
    const int vec = C % 8 == 0 ? 8 : 1, G = C / vec;
    PCNN_REQUIRE((long)H * W * C <= INT32_MAX - POOL_THREADS, PCNN_ERR_ARG,
                 "%s: one %dx%dx%d image exceeds the 32-bit index range (H W C < 2^31 - 256 is required)", fn, H, W, C);
    if (row_pitch == 0) row_pitch = (C + 7) / 8 * 8;
    PCNN_REQUIRE(row_pitch >= C && row_pitch % 8 == 0, PCNN_ERR_ARG,
                 "%s: row_pitch %d: 0 (C rounded up to 8) or a multiple of 8 that is >= C = %d is required", fn, row_pitch, C);
    a->HW = H * W;
    a->C = C;
    a->G = G;
    a->Gc = G < GAP_MAX_GROUPS ? G : GAP_MAX_GROUPS;
    a->slices = (G + a->Gc - 1) / a->Gc;
    a->lanes = POOL_THREADS / a->Gc;
    a->per_cta = GAP_ITERS * a->lanes;
    a->ranges = (a->HW + a->per_cta - 1) / a->per_cta;
    a->pitch = row_pitch;
    a->hw = (double)(float)a->HW;
    a->rhw = 1.0 / a->hw;
    PCNN_REQUIRE((long)N * a->ranges * a->slices <= INT32_MAX && (long)N * ((a->HW * G + POOL_THREADS - 1) / POOL_THREADS) <= INT32_MAX,
                 PCNN_ERR_ARG, "%s: %d images of %dx%dx%d exceed the grid", fn, N, H, W, C);
    return PCNN_OK;
}

extern "C" int pcnn_maxpool_nhwc_info(int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int row_pitch,
                                      int image_rows, int *out5) {
    return pool_info("pcnn_maxpool_nhwc_info", N, H, W, C, R, S, stride, pad_h, pad_w, row_pitch, image_rows, out5);
}

extern "C" int pcnn_avgpool_nhwc_info(int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int row_pitch,
                                      int image_rows, int *out5) {
    return pool_info("pcnn_avgpool_nhwc_info", N, H, W, C, R, S, stride, pad_h, pad_w, row_pitch, image_rows, out5);
}

extern "C" int pcnn_avgpool_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, void *y_bf16_dev, int N, int H, int W, int C, int R, int S,
                                          int stride, int pad_h, int pad_w, int count_include_pad, int y_row_pitch, int y_image_rows) {
    const char *fn = "pcnn_avgpool_nhwc_bf16_fwd";
    PCNN_REQUIRE(ctx && x_bf16_dev && y_bf16_dev, PCNN_ERR_ARG, "%s: NULL context, x or y", fn);
    int rc = include_pad_flag(fn, count_include_pad);
    if (rc) return rc;
    PoolShape sh;
    if ((rc = pool_shape(fn, N, H, W, C, R, S, stride, pad_h, pad_w, y_row_pitch, y_image_rows, &sh))) return rc;
    PoolArgs &a = sh.args;
    PCNN_REQUIRE(aligned16(x_bf16_dev) && aligned16(y_bf16_dev), PCNN_ERR_ARG, "%s: x and y must be 16-byte aligned", fn);
    const size_t xb = (size_t)N * H * W * C * 2, yb = (size_t)N * a.rows * a.pitch * 2;
    PCNN_REQUIRE(!overlap(x_bf16_dev, xb, y_bf16_dev, yb), PCNN_ERR_ARG, "%s: overlapping buffers: x and y must not share memory", fn);
    unsigned grid;
    if ((rc = pool_grid(fn, N, &a, a.P * a.Q * a.G, &grid))) return rc;
    pcnn_device_guard dg(ctx->device);
    const auto *x = static_cast<const __nv_bfloat16 *>(x_bf16_dev);
    auto *y = static_cast<__nv_bfloat16 *>(y_bf16_dev);
    if (sh.vec == 8)
        k_avgpool_nhwc_fwd<8><<<grid, POOL_THREADS, 0, ctx->stream>>>(x, y, a, count_include_pad);
    else
        k_avgpool_nhwc_fwd<1><<<grid, POOL_THREADS, 0, ctx->stream>>>(x, y, a, count_include_pad);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_avgpool_nhwc_bf16_bwd(pcnn_ctx *ctx, const void *dy_bf16_dev, void *dx_bf16_dev, int N, int H, int W, int C, int R, int S,
                                          int stride, int pad_h, int pad_w, int count_include_pad, int dy_row_pitch, int dy_image_rows) {
    const char *fn = "pcnn_avgpool_nhwc_bf16_bwd";
    PCNN_REQUIRE(ctx && dy_bf16_dev && dx_bf16_dev, PCNN_ERR_ARG, "%s: NULL context, dy or dx", fn);
    int rc = include_pad_flag(fn, count_include_pad);
    if (rc) return rc;
    PoolShape sh;
    if ((rc = pool_shape(fn, N, H, W, C, R, S, stride, pad_h, pad_w, dy_row_pitch, dy_image_rows, &sh))) return rc;
    PoolArgs &a = sh.args;
    PCNN_REQUIRE(aligned16(dy_bf16_dev) && aligned16(dx_bf16_dev), PCNN_ERR_ARG, "%s: dy and dx must be 16-byte aligned", fn);
    const size_t xb = (size_t)N * H * W * C * 2, yb = (size_t)N * a.rows * a.pitch * 2;
    PCNN_REQUIRE(!overlap(dx_bf16_dev, xb, dy_bf16_dev, yb), PCNN_ERR_ARG, "%s: overlapping buffers: dy and dx must not share memory", fn);
    unsigned grid;
    if ((rc = pool_grid(fn, N, &a, H * W * a.G, &grid))) return rc;
    pcnn_device_guard dg(ctx->device);
    const auto *dy = static_cast<const __nv_bfloat16 *>(dy_bf16_dev);
    auto *dx = static_cast<__nv_bfloat16 *>(dx_bf16_dev);
    if (sh.vec == 8)
        k_avgpool_nhwc_bwd<8><<<grid, POOL_THREADS, 0, ctx->stream>>>(dy, dx, a, count_include_pad);
    else
        k_avgpool_nhwc_bwd<1><<<grid, POOL_THREADS, 0, ctx->stream>>>(dy, dx, a, count_include_pad);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_global_avgpool_nhwc_info(int N, int H, int W, int C, int row_pitch, int *out8) {
    const char *fn = "pcnn_global_avgpool_nhwc_info";
    PCNN_REQUIRE(out8, PCNN_ERR_ARG, "%s: NULL out8", fn);
    GapArgs a;
    int rc = gap_shape(fn, N, H, W, C, row_pitch, &a);
    if (rc) return rc;
    out8[0] = a.pitch;
    out8[1] = C / a.G;
    out8[2] = a.Gc;
    out8[3] = a.slices;
    out8[4] = a.lanes;
    out8[5] = a.per_cta;
    out8[6] = a.ranges;
    out8[7] = N * a.ranges * a.slices;
    return PCNN_OK;
}

extern "C" int pcnn_global_avgpool_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, void *y_bf16_dev, int N, int H, int W, int C,
                                                 int y_row_pitch) {
    const char *fn = "pcnn_global_avgpool_nhwc_bf16_fwd";
    PCNN_REQUIRE(ctx && x_bf16_dev && y_bf16_dev, PCNN_ERR_ARG, "%s: NULL context, x or y", fn);
    GapArgs a;
    int rc = gap_shape(fn, N, H, W, C, y_row_pitch, &a);
    if (rc) return rc;
    PCNN_REQUIRE(aligned16(x_bf16_dev) && aligned16(y_bf16_dev), PCNN_ERR_ARG, "%s: x and y must be 16-byte aligned", fn);
    const size_t xb = (size_t)N * a.HW * C * 2, yb = (size_t)N * a.pitch * 2;
    PCNN_REQUIRE(!overlap(x_bf16_dev, xb, y_bf16_dev, yb), PCNN_ERR_ARG, "%s: overlapping buffers: x and y must not share memory", fn);
    pcnn_device_guard dg(ctx->device);
    float *slots = nullptr;
    if (a.ranges > 1 && (rc = pcnn_scratch(ctx, (size_t)N * a.ranges * C * sizeof(float), (void **)&slots))) return rc;
    const auto *x = static_cast<const __nv_bfloat16 *>(x_bf16_dev);
    auto *y = static_cast<__nv_bfloat16 *>(y_bf16_dev);
    const unsigned grid = (unsigned)((long)N * a.ranges * a.slices);
    if (C / a.G == 8)
        k_gap_fwd<8><<<grid, POOL_THREADS, 0, ctx->stream>>>(x, y, slots, a);
    else
        k_gap_fwd<1><<<grid, POOL_THREADS, 0, ctx->stream>>>(x, y, slots, a);
    PCNN_CHECK_LAUNCH(ctx);
    if (a.ranges > 1) {
        k_gap_finish<<<(unsigned)(((long)N * C + POOL_THREADS - 1) / POOL_THREADS), POOL_THREADS, 0, ctx->stream>>>(slots, y, N, a);
        PCNN_CHECK_LAUNCH(ctx);
    }
    return PCNN_OK;
}

extern "C" int pcnn_global_avgpool_nhwc_bf16_bwd(pcnn_ctx *ctx, const void *dy_bf16_dev, void *dx_bf16_dev, int N, int H, int W, int C,
                                                 int dy_row_pitch) {
    const char *fn = "pcnn_global_avgpool_nhwc_bf16_bwd";
    PCNN_REQUIRE(ctx && dy_bf16_dev && dx_bf16_dev, PCNN_ERR_ARG, "%s: NULL context, dy or dx", fn);
    GapArgs a;
    int rc = gap_shape(fn, N, H, W, C, dy_row_pitch, &a);
    if (rc) return rc;
    PCNN_REQUIRE(aligned16(dy_bf16_dev) && aligned16(dx_bf16_dev), PCNN_ERR_ARG, "%s: dy and dx must be 16-byte aligned", fn);
    const size_t xb = (size_t)N * a.HW * C * 2, yb = (size_t)N * a.pitch * 2;
    PCNN_REQUIRE(!overlap(dx_bf16_dev, xb, dy_bf16_dev, yb), PCNN_ERR_ARG, "%s: overlapping buffers: dy and dx must not share memory", fn);
    pcnn_device_guard dg(ctx->device);
    const int blocks = (a.HW * a.G + POOL_THREADS - 1) / POOL_THREADS;
    const unsigned grid = (unsigned)((long)N * blocks);
    const auto *dy = static_cast<const __nv_bfloat16 *>(dy_bf16_dev);
    auto *dx = static_cast<__nv_bfloat16 *>(dx_bf16_dev);
    if (C / a.G == 8)
        k_gap_bwd<8><<<grid, POOL_THREADS, 0, ctx->stream>>>(dy, dx, a, blocks);
    else
        k_gap_bwd<1><<<grid, POOL_THREADS, 0, ctx->stream>>>(dy, dx, a, blocks);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_maxpool_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, void *y_bf16_dev, uint8_t *argmax_dev, int N, int H, int W,
                                          int C, int R, int S, int stride, int pad_h, int pad_w, int y_row_pitch, int y_image_rows) {
    const char *fn = "pcnn_maxpool_nhwc_bf16_fwd";
    PCNN_REQUIRE(ctx && x_bf16_dev && y_bf16_dev, PCNN_ERR_ARG, "%s: NULL context, x or y (argmax alone may be NULL)", fn);
    PoolShape sh;
    int rc = pool_shape(fn, N, H, W, C, R, S, stride, pad_h, pad_w, y_row_pitch, y_image_rows, &sh);
    if (rc) return rc;
    PoolArgs &a = sh.args;
    PCNN_REQUIRE(aligned16(x_bf16_dev) && aligned16(y_bf16_dev) && aligned16(argmax_dev), PCNN_ERR_ARG,
                 "%s: x, y and argmax must be 16-byte aligned", fn);
    const size_t xb = (size_t)N * H * W * C * 2, yb = (size_t)N * a.rows * a.pitch * 2, ab = (size_t)N * a.P * a.Q * C;
    PCNN_REQUIRE(!overlap(x_bf16_dev, xb, y_bf16_dev, yb) && !overlap(x_bf16_dev, xb, argmax_dev, ab) &&
                     !overlap(y_bf16_dev, yb, argmax_dev, ab),
                 PCNN_ERR_ARG, "%s: overlapping buffers: x, y and argmax must not share memory", fn);
    unsigned grid;
    rc = pool_grid(fn, N, &a, a.P * a.Q * a.G, &grid);
    if (rc) return rc;
    pcnn_device_guard dg(ctx->device);
    const auto *x = static_cast<const __nv_bfloat16 *>(x_bf16_dev);
    auto *y = static_cast<__nv_bfloat16 *>(y_bf16_dev);
    if (sh.vec == 8)
        k_maxpool_nhwc_fwd<8><<<grid, POOL_THREADS, 0, ctx->stream>>>(x, y, argmax_dev, a);
    else
        k_maxpool_nhwc_fwd<1><<<grid, POOL_THREADS, 0, ctx->stream>>>(x, y, argmax_dev, a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_maxpool_nhwc_bf16_bwd(pcnn_ctx *ctx, const void *dy_bf16_dev, const uint8_t *argmax_dev, void *dx_bf16_dev, int N, int H,
                                          int W, int C, int R, int S, int stride, int pad_h, int pad_w, int dy_row_pitch, int dy_image_rows) {
    const char *fn = "pcnn_maxpool_nhwc_bf16_bwd";
    PCNN_REQUIRE(ctx && dy_bf16_dev && argmax_dev && dx_bf16_dev, PCNN_ERR_ARG, "%s: NULL context, dy, argmax or dx", fn);
    PoolShape sh;
    int rc = pool_shape(fn, N, H, W, C, R, S, stride, pad_h, pad_w, dy_row_pitch, dy_image_rows, &sh);
    if (rc) return rc;
    PoolArgs &a = sh.args;
    PCNN_REQUIRE(aligned16(dy_bf16_dev) && aligned16(argmax_dev) && aligned16(dx_bf16_dev), PCNN_ERR_ARG,
                 "%s: dy, argmax and dx must be 16-byte aligned", fn);
    const size_t xb = (size_t)N * H * W * C * 2, yb = (size_t)N * a.rows * a.pitch * 2, ab = (size_t)N * a.P * a.Q * C;
    PCNN_REQUIRE(!overlap(dx_bf16_dev, xb, dy_bf16_dev, yb) && !overlap(dx_bf16_dev, xb, argmax_dev, ab), PCNN_ERR_ARG,
                 "%s: overlapping buffers: dy and argmax must not share memory with dx", fn);
    unsigned grid;
    rc = pool_grid(fn, N, &a, H * W * a.G, &grid);
    if (rc) return rc;
    pcnn_device_guard dg(ctx->device);
    const auto *dy = static_cast<const __nv_bfloat16 *>(dy_bf16_dev);
    auto *dx = static_cast<__nv_bfloat16 *>(dx_bf16_dev);
    if (sh.vec == 8)
        k_maxpool_nhwc_bwd<8><<<grid, POOL_THREADS, 0, ctx->stream>>>(dy, argmax_dev, dx, a);
    else
        k_maxpool_nhwc_bwd<1><<<grid, POOL_THREADS, 0, ctx->stream>>>(dy, argmax_dev, dx, a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
