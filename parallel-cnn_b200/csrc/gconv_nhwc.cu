// parallel-cnn_b200/csrc/gconv_nhwc.cu -- grouped convolution (groups = G, 1 < G < C: each group of Cg = C / G input channels feeds
// its own Kg = K / G filters) between bf16 NHWC layers: pcnn_gconv_plan_create (a pcnn_conv_plan run by pcnn_conv_tc_fwd, refreshed
// by pcnn_conv_plan_set_params and the optimizer), pcnn_gconv_wgrad, pcnn_gconv_dgrad and pcnn_gconv_info.  The contract is in
// include/pcnn.h.
//
// All three passes run fp32 FMAs on the CUDA cores in the order pcnn.h states.  Each pass moves 16-byte vectors of 8 channels along
// its reduced channel axis when that axis has a multiple of 8 channels, otherwise vectors of 4, 2 or 1 (the largest that divides it);
// and each thread owns a tile of 8, 4, 2 or 1 output channels of one group (the largest that divides the group's width), so every
// loaded activation feeds a tile of filters and every staged filter value feeds several pixels.
//   - Forward: CTA (strip block, k slice) stages the bf16 filters of its output channels, [K][R][S][Cg] in the plan, through shared
//     memory as [r][s][c][k]; thread (strip, k tile) computes KT channels at GC_PX consecutive q of one output row.
//   - Input gradient: a gather like the depthwise one.  CTA (strip block, c slice) stages w[g Kg + k][r][s][c] of its input channels
//     as [r][s][k][c]; thread (strip, c tile) owns CT channels at GC_PX consecutive w of one input row, visits the dy rows on the
//     stride grid in ascending r, then s, then k, and writes every dx element once, with no memset and no atomics.
//   - Weight gradient: CTA (pixel range, item block); an item is (k tile, tap, c vector).  Each thread keeps KT x VEC fp32 sums over
//     the pixels lane, lane + lanes, ... of its range, the lanes are added in lane order through shared memory, and each range writes
//     an fp32 slot [K][R][S][Cg] that pcnn_conv_wgrad_reduce_slots adds in a fixed order.  The ranges depend on the shape only.
#include "pcnn_internal.h"

#include <cuda_bf16.h>

#include <algorithm>
#include <memory>

namespace {

constexpr int GC_THREADS = 256;
constexpr int GC_SMEM_ELEMS = 36864;      // bf16 filter elements a CTA stages (72 KiB), and the limit on one group's Kg Cg R S
constexpr int GC_MAX_WIDTH = 32;          // channel tiles per CTA of the forward and the input gradient
constexpr int GC_PX = 4;                  // outputs (forward) or dx elements (input gradient) per thread along a row
constexpr int GC_WG_ITEMS = 32;           // weight-gradient items per CTA (one warp's width)
constexpr int GC_WG_LANES = GC_THREADS / GC_WG_ITEMS;
constexpr int GC_WG_ITERS = 64;           // pixels per lane of the weight gradient

template <int VEC>
struct alignas(2 * VEC) BfVec {
    __nv_bfloat16 h[VEC];
};

template <int VEC>
__device__ __forceinline__ BfVec<VEC> bf_zero() {
    BfVec<VEC> v;
#pragma unroll
    for (int c = 0; c < VEC; ++c) v.h[c] = __ushort_as_bfloat16(0);
    return v;
}

struct GcArgs {
    int N, H, W, C, K, G, Cg, Kg, R, S, stride, pad_h, pad_w, P, Q;
    int RSC;                    // R S Cg: one filter
    int vc, vk;                 // vector / tile widths along Cg and Kg: the largest of 8, 4, 2, 1 dividing each
    int fw, fslices, flanes;    // forward: k tiles (of vk) per CTA, k slices, strips per CTA
    int dwid, dslices, dlanes;  // input gradient: c tiles (of vc) per CTA, c slices, strips per CTA
    int qb, wb;                 // strips per output row (forward) and per input row (input gradient)
    long long fstrips, dstrips; // N P qb, N H wb
    long long M;                // N P Q output pixels
    int items, iblocks;         // weight gradient: (k tile, tap, c vector) items and blocks of GC_WG_ITEMS
    int per_range, ranges;      // weight gradient: pixels per range and ranges
    int act;
};

// forward: y[n][p][q][k] for the KT channels k.. of one group at GC_PX consecutive q; VEC channels of x per load
template <int VEC, int KT>
__global__ void __launch_bounds__(GC_THREADS) k_gconv_fwd(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ wop,
                                                          const float *__restrict__ bias, __nv_bfloat16 *__restrict__ y, GcArgs a) {
    extern __shared__ __align__(16) __nv_bfloat16 wsm[];    // [r][s][c][width]: the slice's filters, KT channels of a tile adjacent
    const int width = a.fw * KT, k0 = blockIdx.y * width, nk = min(width, a.K - k0);
    for (int i = threadIdx.x; i < nk * a.RSC; i += GC_THREADS) {
        const int kl = i / a.RSC;
        wsm[(i - kl * a.RSC) * width + kl] = wop[(long)k0 * a.RSC + i];
    }
    __syncthreads();
    const int j = threadIdx.x % a.fw, lane = threadIdx.x / a.fw;
    const long long strip = (long long)blockIdx.x * a.flanes + lane;
    if (lane >= a.flanes || j * KT >= nk || strip >= a.fstrips) return;
    const int n = (int)(strip / ((long long)a.P * a.qb));
    const int rem = (int)(strip - (long long)n * a.P * a.qb), p = rem / a.qb, q0 = (rem - p * a.qb) * GC_PX;
    const int k = k0 + j * KT, st = a.stride;
    const __nv_bfloat16 *xi = x + (long)n * a.H * a.W * a.C + (k / a.Kg) * a.Cg;
    const __nv_bfloat16 *wt = wsm + j * KT;
    float acc[GC_PX][KT];                                  // -0 + t == t for every t: each sum starts from its first term
#pragma unroll
    for (int i = 0; i < GC_PX; ++i)
#pragma unroll
        for (int kk = 0; kk < KT; ++kk) acc[i][kk] = -0.0f;
    for (int r = 0; r < a.R; ++r) {
        const int h = p * st - a.pad_h + r;
        const bool rowok = h >= 0 && h < a.H;
        const __nv_bfloat16 *row = xi + (long)h * a.W * a.C;
        for (int s = 0; s < a.S; ++s) {
            const __nv_bfloat16 *wtap = wt + (r * a.S + s) * a.Cg * width;
            for (int c0 = 0; c0 < a.Cg; c0 += VEC) {
                BfVec<VEC> xv[GC_PX];
#pragma unroll
                for (int i = 0; i < GC_PX; ++i) {
                    const int w = (q0 + i) * st - a.pad_w + s;
                    xv[i] = rowok && w >= 0 && w < a.W ? *reinterpret_cast<const BfVec<VEC> *>(row + (long)w * a.C + c0) : bf_zero<VEC>();
                }
#pragma unroll
                for (int e = 0; e < VEC; ++e) {
                    const BfVec<KT> wv = *reinterpret_cast<const BfVec<KT> *>(wtap + (c0 + e) * width);
#pragma unroll
                    for (int i = 0; i < GC_PX; ++i)
#pragma unroll
                        for (int kk = 0; kk < KT; ++kk)
                            acc[i][kk] = fmaf(__bfloat162float(xv[i].h[e]), __bfloat162float(wv.h[kk]), acc[i][kk]);
                }
            }
        }
    }
    __nv_bfloat16 *yo = y + (((long)n * a.P + p) * a.Q + q0) * a.K + k;
#pragma unroll
    for (int i = 0; i < GC_PX; ++i) {
        if (q0 + i >= a.Q) break;
        BfVec<KT> out;
#pragma unroll
        for (int kk = 0; kk < KT; ++kk) {
            float v = bias ? __fadd_rn(acc[i][kk], bias[k + kk]) : acc[i][kk];
            if (a.act == PCNN_ACT_RELU) v = v < 0.0f ? 0.0f : v;
            out.h[kk] = __float2bfloat16_rn(v);
        }
        *reinterpret_cast<BfVec<KT> *>(yo + (long)i * a.K) = out;
    }
}

// input gradient: dx[n][h][w][c] for the CT channels c.. of one group at GC_PX consecutive w; VEC channels of dy per load
template <int VEC, int CT>
__global__ void __launch_bounds__(GC_THREADS, 2) k_gconv_dgrad(const __nv_bfloat16 *__restrict__ dy, const __nv_bfloat16 *__restrict__ wop,
                                                            __nv_bfloat16 *__restrict__ dx, GcArgs a) {
    extern __shared__ __align__(16) __nv_bfloat16 wsm[];    // [r][s][k][width]: w[g Kg + k][r][s][c] for the slice's channels c
    const int width = a.dwid * CT, c0 = blockIdx.y * width, nc = min(width, a.C - c0), RS = a.R * a.S;
    for (int i = threadIdx.x; i < nc * RS * a.Kg; i += GC_THREADS) {
        const int cl = i % nc, tk = i / nc, t = tk / a.Kg, k = tk - t * a.Kg;
        const int c = c0 + cl, g = c / a.Cg;
        wsm[tk * width + cl] = wop[((long)(g * a.Kg + k) * RS + t) * a.Cg + (c - g * a.Cg)];
    }
    __syncthreads();
    const int j = threadIdx.x % a.dwid, lane = threadIdx.x / a.dwid;
    const long long strip = (long long)blockIdx.x * a.dlanes + lane;
    if (lane >= a.dlanes || j * CT >= nc || strip >= a.dstrips) return;
    const int n = (int)(strip / ((long long)a.H * a.wb));
    const int rem = (int)(strip - (long long)n * a.H * a.wb), h = rem / a.wb, w0 = (rem - h * a.wb) * GC_PX;
    const int c = c0 + j * CT, st = a.stride;
    const __nv_bfloat16 *dyi = dy + (long)n * a.P * a.Q * a.K + (c / a.Cg) * a.Kg;
    const __nv_bfloat16 *wt = wsm + j * CT;
    float acc[GC_PX][CT];
#pragma unroll
    for (int i = 0; i < GC_PX; ++i)
#pragma unroll
        for (int cc = 0; cc < CT; ++cc) acc[i][cc] = -0.0f;
    bool hit[GC_PX];
#pragma unroll
    for (int i = 0; i < GC_PX; ++i) hit[i] = false;
    for (int r = 0; r < a.R; ++r) {
        const int t = h + a.pad_h - r;
        if (t < 0 || t % st != 0 || t / st >= a.P) continue;
        const __nv_bfloat16 *row = dyi + (long)(t / st) * a.Q * a.K;
        for (int s = 0; s < a.S; ++s) {
            int qo[GC_PX];                                 // offset of the dy pixel of dx element i at tap (r, s), -1 for none
            bool any = false;
#pragma unroll
            for (int i = 0; i < GC_PX; ++i) {
                const int u = w0 + i + a.pad_w - s;
                const bool ok = w0 + i < a.W && u >= 0 && u % st == 0 && u / st < a.Q;
                qo[i] = ok ? u / st * a.K : -1;
                hit[i] = hit[i] || ok;
                any = any || ok;
            }
            if (!any) continue;
            const __nv_bfloat16 *wtap = wt + (r * a.S + s) * a.Kg * width;
            for (int k0 = 0; k0 < a.Kg; k0 += VEC) {
                BfVec<VEC> dv[GC_PX];
#pragma unroll
                for (int i = 0; i < GC_PX; ++i)
                    dv[i] = qo[i] >= 0 ? *reinterpret_cast<const BfVec<VEC> *>(row + qo[i] + k0) : bf_zero<VEC>();
#pragma unroll
                for (int e = 0; e < VEC; ++e) {
                    const BfVec<CT> wv = *reinterpret_cast<const BfVec<CT> *>(wtap + (k0 + e) * width);
#pragma unroll
                    for (int i = 0; i < GC_PX; ++i) {
                        if (qo[i] < 0) continue;
#pragma unroll
                        for (int cc = 0; cc < CT; ++cc)
                            acc[i][cc] = fmaf(__bfloat162float(dv[i].h[e]), __bfloat162float(wv.h[cc]), acc[i][cc]);
                    }
                }
            }
        }
    }
    __nv_bfloat16 *dxo = dx + (((long)n * a.H + h) * a.W + w0) * a.C + c;
#pragma unroll
    for (int i = 0; i < GC_PX; ++i) {
        if (w0 + i >= a.W) break;
        BfVec<CT> out;
#pragma unroll
        for (int cc = 0; cc < CT; ++cc) out.h[cc] = hit[i] ? __float2bfloat16_rn(acc[i][cc]) : __ushort_as_bfloat16(0);
        *reinterpret_cast<BfVec<CT> *>(dxo + (long)i * a.C) = out;
    }
}

// CTA (range, item block): out[k][r][s][c] for the block's items over the pixels [range * per_range, (range + 1) * per_range) of
// the N P Q output pixels; `out` is dw itself when there is one range, otherwise slot `range` of the [ranges][K][R][S][Cg] partials.
// Item i is (k tile i / (R S Cg / VEC), tap, c vector), the c vector fastest.
template <int VEC, int KT>
__global__ void __launch_bounds__(GC_THREADS) k_gconv_wgrad(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ dy,
                                                            float *__restrict__ out, GcArgs a) {
    __shared__ float part[GC_WG_LANES][GC_WG_ITEMS * VEC];
    const int il = threadIdx.x % GC_WG_ITEMS, lane = threadIdx.x / GC_WG_ITEMS;
    const int per_k = a.RSC / VEC;
    auto decode = [&](int item, int *k, int *t, int *cv) {
        const int kt = item / per_k, rest = item - kt * per_k;
        *k = kt * KT;
        *t = rest / (a.Cg / VEC);
        *cv = (rest - *t * (a.Cg / VEC)) * VEC;
    };
    const int item = blockIdx.y * GC_WG_ITEMS + il;
    const bool on = item < a.items;
    const long long p0 = (long long)blockIdx.x * a.per_range;
    const int active = (int)min((long long)GC_WG_LANES, a.M - p0);   // lanes holding at least one pixel
    float acc[KT][VEC];
#pragma unroll
    for (int kk = 0; kk < KT; ++kk)
#pragma unroll
        for (int e = 0; e < VEC; ++e) acc[kk][e] = -0.0f;
    if (on) {
        int k, t, cv;
        decode(item, &k, &t, &cv);
        const int r = t / a.S, s = t - r * a.S, st = a.stride, PQ = a.P * a.Q;
        const int c = (k / a.Kg) * a.Cg + cv;
        for (int i = 0; i < GC_WG_ITERS; ++i) {
            const long long m = p0 + lane + (long long)i * GC_WG_LANES;
            if (m >= a.M) break;
            const int n = (int)(m / PQ), pq = (int)(m - (long long)n * PQ), p = pq / a.Q, q = pq - p * a.Q;
            const BfVec<KT> d = *reinterpret_cast<const BfVec<KT> *>(dy + m * a.K + k);
            const int h = p * st - a.pad_h + r, w = q * st - a.pad_w + s;
            BfVec<VEC> xv = bf_zero<VEC>();
            if (h >= 0 && h < a.H && w >= 0 && w < a.W) xv = *reinterpret_cast<const BfVec<VEC> *>(x + (((long)n * a.H + h) * a.W + w) * a.C + c);
#pragma unroll
            for (int kk = 0; kk < KT; ++kk)
#pragma unroll
                for (int e = 0; e < VEC; ++e) acc[kk][e] = fmaf(__bfloat162float(d.h[kk]), __bfloat162float(xv.h[e]), acc[kk][e]);
        }
    }
    float *slot = out + (long)blockIdx.x * a.K * a.RSC;
#pragma unroll
    for (int kk = 0; kk < KT; ++kk) {
#pragma unroll
        for (int e = 0; e < VEC; ++e) part[lane][il * VEC + e] = acc[kk][e];
        __syncthreads();
        for (int o = threadIdx.x; o < GC_WG_ITEMS * VEC; o += GC_THREADS) {
            const int oi = blockIdx.y * GC_WG_ITEMS + o / VEC;
            if (oi >= a.items) continue;
            float v = part[0][o];
            for (int l = 1; l < active; ++l) v = __fadd_rn(v, part[l][o]);
            int k, t, cv;
            decode(oi, &k, &t, &cv);
            slot[(long)(k + kk) * a.RSC + t * a.Cg + cv + o % VEC] = v;
        }
        __syncthreads();
    }
}

int vec_of(int n) { return n % 8 == 0 ? 8 : n % 4 == 0 ? 4 : n % 2 == 0 ? 2 : 1; }

// the domain of pcnn.h, refused with PCNN_ERR_ARG and a message naming `fn`, and the partition, a function of the shape alone
int gc_shape(const char *fn, int N, int H, int W, int C, int K, int G, int R, int S, int stride, int pad_h, int pad_w, GcArgs *a) {
    int P, Q;
    int rc = nhwc_window_check(fn, N, H, W, C, R, S, stride, pad_h, pad_w, &P, &Q);
    if (rc) return rc;
    PCNN_REQUIRE(K >= 1, PCNN_ERR_ARG, "%s: K = %d: K >= 1 is required", fn, K);
    PCNN_REQUIRE(G != 1, PCNN_ERR_ARG,
                 "%s: groups = 1 is a dense convolution: use ConvLayer (pcnn_conv_tc_plan_create_strided or pcnn_conv_wide_plan_create)", fn);
    PCNN_REQUIRE(G >= 2, PCNN_ERR_ARG, "%s: groups = %d: G >= 2 is required", fn, G);
    PCNN_REQUIRE(C % G == 0 && K % G == 0, PCNN_ERR_ARG, "%s: C = %d, K = %d, groups = %d: C %% G == 0 and K %% G == 0 are required", fn,
                 C, K, G);
    const int Cg = C / G, Kg = K / G;
    PCNN_REQUIRE(!(Cg == 1 && Kg == 1), PCNN_ERR_ARG,
                 "%s: groups = C = K is a depthwise convolution: use pcnn_dwconv_plan_create (DepthwiseConvLayer)", fn);
    PCNN_REQUIRE((long)Kg * Cg * R * S <= GC_SMEM_ELEMS, PCNN_ERR_ARG,
                 "%s: one group's filters Kg Cg R S = %d x %d x %d x %d exceed %d: Kg Cg R S <= %d is required (shared-memory staging)", fn,
                 Kg, Cg, R, S, GC_SMEM_ELEMS, GC_SMEM_ELEMS);
    PCNN_REQUIRE((long)H * W * C <= INT32_MAX && (long)P * Q * K <= INT32_MAX && (long)K * R * S * Cg <= INT32_MAX, PCNN_ERR_ARG,
                 "%s: one %dx%dx%d image, its %dx%dx%d output or its %d x %d x %d x %d filters exceed the 32-bit index range: H W C, P Q K and "
                 "K R S Cg < 2^31 are required", fn, H, W, C, P, Q, K, K, R, S, Cg);
    GcArgs &g = *a;
    g.N = N; g.H = H; g.W = W; g.C = C; g.K = K; g.G = G; g.Cg = Cg; g.Kg = Kg; g.R = R; g.S = S; g.stride = stride;
    g.pad_h = pad_h; g.pad_w = pad_w; g.P = P; g.Q = Q;
    g.RSC = R * S * Cg;
    g.vc = vec_of(Cg);
    g.vk = vec_of(Kg);
    const int ktiles = K / g.vk, ctiles = C / g.vc;
    g.fw = std::min(std::min(GC_MAX_WIDTH, ktiles), GC_SMEM_ELEMS / (g.vk * g.RSC));
    g.fslices = (ktiles + g.fw - 1) / g.fw;
    g.flanes = GC_THREADS / g.fw;
    g.dwid = std::min(std::min(GC_MAX_WIDTH, ctiles), GC_SMEM_ELEMS / (g.vc * R * S * Kg));
    g.dslices = (ctiles + g.dwid - 1) / g.dwid;
    g.dlanes = GC_THREADS / g.dwid;
    g.qb = (Q + GC_PX - 1) / GC_PX;
    g.wb = (W + GC_PX - 1) / GC_PX;
    g.fstrips = (long long)N * P * g.qb;
    g.dstrips = (long long)N * H * g.wb;
    g.M = (long long)N * P * Q;
    g.items = (K / g.vk) * (g.RSC / g.vc);
    g.iblocks = (g.items + GC_WG_ITEMS - 1) / GC_WG_ITEMS;
    g.per_range = GC_WG_LANES * GC_WG_ITERS;
    const long long ranges = (g.M + g.per_range - 1) / g.per_range;
    PCNN_REQUIRE(g.fslices <= 65535 && g.dslices <= 65535 && g.iblocks <= 65535 && ranges <= INT32_MAX &&
                     (g.fstrips + g.flanes - 1) / g.flanes <= INT32_MAX && (g.dstrips + g.dlanes - 1) / g.dlanes <= INT32_MAX,
                 PCNN_ERR_ARG, "%s: %d images of %dx%dx%d with K = %d exceed the grid", fn, N, H, W, C, K);
    g.ranges = (int)ranges;
    g.act = 0;
    return PCNN_OK;
}

// additions on the longest path of one weight-gradient sum: the pixels of a lane, the lanes of a range, then (with several
// ranges) pcnn_conv_wgrad_reduce_slots: every 8th slot added to +0, then a tree over the 8
int gc_n_acc(const GcArgs &a) {
    const int lane_px = a.M < a.per_range ? (int)((a.M + GC_WG_LANES - 1) / GC_WG_LANES) : GC_WG_ITERS;
    const int lanes = (int)(a.M < GC_WG_LANES ? a.M : GC_WG_LANES);
    return (lane_px - 1) + (lanes - 1) + (a.ranges > 1 ? (a.ranges + 7) / 8 + 3 : 0);
}

bool overlap(const void *p, size_t np, const void *q, size_t nq) {
    const uintptr_t a = (uintptr_t)p, b = (uintptr_t)q;
    return a < b + nq && b < a + np;
}

bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

typedef void (*pass_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, const float *, __nv_bfloat16 *, GcArgs);
typedef void (*dgrad_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, __nv_bfloat16 *, GcArgs);
typedef void (*wgrad_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, float *, GcArgs);

int log2_of(int v) { return v == 8 ? 3 : v == 4 ? 2 : v == 2 ? 1 : 0; }

#define GC_TABLE(kern, V)                                                                                                       \
    { kern<V, 1>, kern<V, 2>, kern<V, 4>, kern<V, 8> }
#define GC_TABLES(kern) { GC_TABLE(kern, 1), GC_TABLE(kern, 2), GC_TABLE(kern, 4), GC_TABLE(kern, 8) }

const pass_fn fwd_table[4][4] = GC_TABLES(k_gconv_fwd);
const dgrad_fn dgrad_table[4][4] = GC_TABLES(k_gconv_dgrad);
const wgrad_fn wgrad_table[4][4] = GC_TABLES(k_gconv_wgrad);

// a launch with more than the default 48 KiB of dynamic shared memory needs the kernel's opt-in
int smem_opt_in(const void *k, size_t bytes) {
    if (bytes > 48 * 1024) PCNN_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return PCNN_OK;
}

}  // namespace

// a plan of pcnn_gconv_plan_create: w is [K][R][S][Cg], the fp32 master's element order (one row of n elements)
struct GConvPlan : pcnn_conv_plan {
    static constexpr const char *made_by = "pcnn_gconv_plan_create";
    GcArgs a;
    const __nv_bfloat16 *wop() const { return static_cast<const __nv_bfloat16 *>(w); }
    int fwd(pcnn_ctx *ctx, const void *x_bf16, void *y_bf16) override;
};

extern "C" int pcnn_gconv_info(int N, int H, int W, int C, int K, int G, int R, int S, int stride, int pad_h, int pad_w, int *out16) {
    const char *fn = "pcnn_gconv_info";
    PCNN_REQUIRE(out16, PCNN_ERR_ARG, "%s: NULL out16", fn);
    GcArgs a;
    int rc = gc_shape(fn, N, H, W, C, K, G, R, S, stride, pad_h, pad_w, &a);
    if (rc) return rc;
    const int v[16] = {a.P,     a.Q,    a.Cg,      a.Kg,     a.vc,      a.vk,       a.fw,        a.fslices,
                       a.dwid,  a.dslices, a.items, a.iblocks, a.per_range, a.ranges, gc_n_acc(a), GC_WG_LANES};
    memcpy(out16, v, sizeof(v));
    return PCNN_OK;
}

extern "C" int pcnn_gconv_plan_create(pcnn_ctx *ctx, int N, int H, int W, int C, int K, int G, int R, int S, int stride, int pad_h,
                                      int pad_w, int act, const float *filt_host, const float *bias_host, pcnn_conv_plan **out) {
    const char *fn = "pcnn_gconv_plan_create";
    PCNN_REQUIRE(ctx && filt_host && out, PCNN_ERR_ARG, "%s: NULL context, filters or out", fn);
    PCNN_REQUIRE_ACT(fn, act);
    PCNN_REQUIRE(act != PCNN_ACT_SIGMOID, PCNN_ERR_ARG,
                 "%s: act 1 (sigmoid) is not supported: the sigmoid of the conv epilogues uses tanh.approx, which no reference can replay "
                 "bit for bit; use act 0 or 3", fn);
    GcArgs a;
    int rc = gc_shape(fn, N, H, W, C, K, G, R, S, stride, pad_h, pad_w, &a);
    if (rc) return rc;
    a.act = act;
    pcnn_device_guard g(ctx->device);
    std::unique_ptr<GConvPlan> pl(new GConvPlan());   // frees a half-built plan on every early return below
    pl->a = a;
    pl->n = (long long)K * a.RSC;
    pl->cols = pl->pitch = (int)pl->n;
    pl->K = K;
    if ((rc = pcnn_plan_upload(ctx, pl.get(), &pl->w, (size_t)pl->n * 2, filt_host, bias_host))) return rc;
    *out = pl.release();
    return PCNN_OK;
}

int GConvPlan::fwd(pcnn_ctx *ctx, const void *x_bf16, void *y_bf16) {
    const char *fn = "pcnn_conv_tc_fwd";
    PCNN_REQUIRE(aligned16(y_bf16), PCNN_ERR_ARG, "%s: the output must be 16-byte aligned", fn);
    const size_t xb = (size_t)a.N * a.H * a.W * a.C * 2, yb = (size_t)a.M * a.K * 2;
    PCNN_REQUIRE(!overlap(x_bf16, xb, y_bf16, yb), PCNN_ERR_ARG, "%s: overlapping buffers: x and y of a grouped plan must not share memory",
                 fn);
    const pass_fn k = fwd_table[log2_of(a.vc)][log2_of(a.vk)];
    const size_t smem = (size_t)a.fw * a.vk * a.RSC * 2;
    int rc = smem_opt_in((const void *)k, smem);
    if (rc) return rc;
    const dim3 grid((unsigned)((a.fstrips + a.flanes - 1) / a.flanes), (unsigned)a.fslices);
    k<<<grid, GC_THREADS, smem, ctx->stream>>>(static_cast<const __nv_bfloat16 *>(x_bf16), wop(), bias,
                                                static_cast<__nv_bfloat16 *>(y_bf16), a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_gconv_wgrad(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *x_bf16, const void *dy_bf16, float *dw_f32) {
    const char *fn = "pcnn_gconv_wgrad";
    PCNN_REQUIRE(ctx && plan && x_bf16 && dy_bf16 && dw_f32, PCNN_ERR_ARG, "%s: NULL argument", fn);
    GConvPlan *pl;
    int rc = plan_as(fn, plan, &pl);
    if (rc) return rc;
    PCNN_REQUIRE(aligned16(x_bf16) && aligned16(dy_bf16) && aligned16(dw_f32), PCNN_ERR_ARG, "%s: x, dy and dw must be 16-byte aligned", fn);
    const GcArgs &a = pl->a;
    const size_t xb = (size_t)a.N * a.H * a.W * a.C * 2, yb = (size_t)a.M * a.K * 2, nout = (size_t)a.K * a.RSC;
    PCNN_REQUIRE(!overlap(dw_f32, nout * 4, x_bf16, xb) && !overlap(dw_f32, nout * 4, dy_bf16, yb), PCNN_ERR_ARG,
                 "%s: overlapping buffers: dw must not share memory with x or dy", fn);
    pcnn_device_guard g(ctx->device);
    float *out = dw_f32;
    if (a.ranges > 1 && (rc = pcnn_scratch(ctx, (size_t)a.ranges * nout * sizeof(float), (void **)&out))) return rc;
    const dim3 grid((unsigned)a.ranges, (unsigned)a.iblocks);
    wgrad_table[log2_of(a.vc)][log2_of(a.vk)]<<<grid, GC_THREADS, 0, ctx->stream>>>(static_cast<const __nv_bfloat16 *>(x_bf16),
                                                                                   static_cast<const __nv_bfloat16 *>(dy_bf16), out, a);
    PCNN_CHECK_LAUNCH(ctx);
    return a.ranges > 1 ? pcnn_conv_wgrad_reduce_slots(ctx, out, dw_f32, a.ranges, (int)nout) : PCNN_OK;
}

extern "C" int pcnn_gconv_dgrad(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *dy_bf16, void *dx_bf16) {
    const char *fn = "pcnn_gconv_dgrad";
    PCNN_REQUIRE(ctx && plan && dy_bf16 && dx_bf16, PCNN_ERR_ARG, "%s: NULL argument", fn);
    GConvPlan *pl;
    int rc = plan_as(fn, plan, &pl);
    if (rc) return rc;
    PCNN_REQUIRE(aligned16(dy_bf16) && aligned16(dx_bf16), PCNN_ERR_ARG, "%s: dy and dx must be 16-byte aligned", fn);
    const GcArgs &a = pl->a;
    const size_t xb = (size_t)a.N * a.H * a.W * a.C * 2, yb = (size_t)a.M * a.K * 2;
    PCNN_REQUIRE(!overlap(dx_bf16, xb, dy_bf16, yb), PCNN_ERR_ARG, "%s: overlapping buffers: dy and dx must not share memory", fn);
    pcnn_device_guard g(ctx->device);
    const dgrad_fn k = dgrad_table[log2_of(a.vk)][log2_of(a.vc)];
    const size_t smem = (size_t)a.dwid * a.vc * a.R * a.S * a.Kg * 2;
    if ((rc = smem_opt_in((const void *)k, smem))) return rc;
    const dim3 grid((unsigned)((a.dstrips + a.dlanes - 1) / a.dlanes), (unsigned)a.dslices);
    k<<<grid, GC_THREADS, smem, ctx->stream>>>(static_cast<const __nv_bfloat16 *>(dy_bf16), pl->wop(), static_cast<__nv_bfloat16 *>(dx_bf16),
                                                a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
