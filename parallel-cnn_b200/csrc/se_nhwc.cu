// parallel-cnn_b200/csrc/se_nhwc.cu -- squeeze-and-excitation channel gating of the dense bf16 NHWC activations the conv forwards
// and batch norm write: y = act(x * s[n][c] (+ r)) (pcnn_se_scale_nhwc_bf16_fwd), the gate's gradient ds[n][c] = sum over the
// pixels of g * x (pcnn_se_scale_nhwc_bf16_bwd_gate) and the input gradient dx = g * s (+ dpool / (H W), the squeeze branch)
// (pcnn_se_scale_nhwc_bf16_bwd_input).  s is what a LinearLayer with O = C writes as y, ds what its backward reads as dy, dpool
// the global average pool's dy: the squeeze branch GAP -> fc -> ReLU -> fc -> sigmoid runs on the existing layers with no copy.
// The contract, every operation in its order, is in include/pcnn.h.
//
// Every pass is HBM-bound.  With C % 8 == 0 a thread moves 16-byte vectors of 8 channels of one pixel, otherwise single
// elements.  The forward and the input gradient are elementwise, one thread per (pixel, channel group) and a run of CTAs per
// image, as the global pool's backward.  The gate gradient writes g and reduces g * x over the pixels of each image in the
// global average pool's partition (gap_shape, pcnn_internal.h), so its sums are ordered exactly as GAP's.  No atomics: the bits
// are the same on every run and every H100.
#include "pcnn_internal.h"
#include "tc_common.cuh"

#include <cuda_bf16.h>

#include <algorithm>

namespace {

constexpr int SE_THREADS = GAP_THREADS;

template <int VEC>
struct alignas(2 * VEC) BfVec {
    __nv_bfloat16 h[VEC];
};

template <int VEC>
__device__ __forceinline__ BfVec<VEC> ld(const __nv_bfloat16 *p) {
    return *reinterpret_cast<const BfVec<VEC> *>(p);
}
template <int VEC>
__device__ __forceinline__ void st(__nv_bfloat16 *p, const BfVec<VEC> &v) {
    *reinterpret_cast<BfVec<VEC> *>(p) = v;
}

// y = bf16_rn(act(RN(float(x) * float(s)) (+ float(r)))); i = pixel * G + group, so the element offset in the image is i * VEC
template <int VEC, int ACT>
__global__ void __launch_bounds__(SE_THREADS) k_se_fwd(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ s,
                                                       const __nv_bfloat16 *__restrict__ r, __nv_bfloat16 *__restrict__ y, GapArgs a,
                                                       int blocks) {
    const int n = blockIdx.x / blocks;
    const int i = (blockIdx.x - n * blocks) * SE_THREADS + threadIdx.x;
    if (i >= a.HW * a.G) return;
    const int g = i % a.G;
    const long off = (long)n * a.HW * a.C + (long)i * VEC;
    const BfVec<VEC> xv = ld<VEC>(x + off);
    const BfVec<VEC> sv = ld<VEC>(s + (long)n * a.C + g * VEC);
    BfVec<VEC> rv;
    if (r) rv = ld<VEC>(r + off);
    BfVec<VEC> out;
#pragma unroll
    for (int c = 0; c < VEC; ++c) {
        float v = __fmul_rn(__bfloat162float(xv.h[c]), __bfloat162float(sv.h[c]));
        if (r) v = __fadd_rn(v, __bfloat162float(rv.h[c]));
        if (ACT == PCNN_ACT_RELU) v = pcnn_tc::relu_f32(v);
        out.h[c] = __float2bfloat16_rn(v);
    }
    st<VEC>(y + off, out);
}

// g = bf16_rn(act'(t)) with t = float(dy) (+ float(dy2)): without dy2 dy's bits pass; at act 3 y <= 0 gives +0 (a NaN y passes),
// the rule of batch norm's backward
template <int ACT>
__device__ __forceinline__ __nv_bfloat16 se_dgrad(__nv_bfloat16 dy, __nv_bfloat16 dy2, bool has_dy2, __nv_bfloat16 y) {
    __nv_bfloat16 g = has_dy2 ? __float2bfloat16_rn(__fadd_rn(__bfloat162float(dy), __bfloat162float(dy2))) : dy;
    if (ACT == PCNN_ACT_RELU && __bfloat162float(y) <= 0.0f) g = __ushort_as_bfloat16((unsigned short)0);
    return g;
}

// The gate gradient in GAP's partition (k_gap_fwd): thread (lane, group) writes g for its pixels and sums RN(float(g) * float(x))
// from its first pixel; the lanes holding a pixel are added in lane order; one range per image writes ds = bf16_rn(sum), more
// write fp32 slots [n][range][C] that k_se_finish adds in range order.  g may be dy: each element is read, then written, by
// the same thread.
template <int VEC, int ACT>
__global__ void __launch_bounds__(SE_THREADS) k_se_gate(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ y,
                                                        const __nv_bfloat16 *dy, const __nv_bfloat16 *__restrict__ dy2, __nv_bfloat16 *g_out,
                                                        __nv_bfloat16 *__restrict__ ds, float *__restrict__ slots, GapArgs a) {
    __shared__ float part[SE_THREADS * 8];                 // [lanes][Gc * VEC]: lanes * Gc <= 256
    constexpr int U = VEC == 8 ? 2 : 4;                    // pixels loaded before any is used
    const int slice = blockIdx.x % a.slices, nr = blockIdx.x / a.slices, rg = nr % a.ranges, n = nr / a.ranges;
    const int lane = threadIdx.x / a.Gc, gl = threadIdx.x % a.Gc, g = slice * a.Gc + gl;
    const int width = a.Gc * VEC, p0 = rg * a.per_cta;
    if (lane < a.lanes && g < a.G && p0 + lane < a.HW) {
        const long base = (long)n * a.HW * a.C + g * VEC;
        float acc[VEC];
        for (int j0 = 0; j0 < GAP_ITERS; j0 += U) {
            BfVec<VEC> xv[U], dv[U], yv[U], d2[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int px = p0 + lane + (j0 + u) * a.lanes;
                if (px < a.HW) {
                    const long off = base + (long)px * a.C;
                    xv[u] = ld<VEC>(x + off);
                    dv[u] = ld<VEC>(dy + off);
                    if (ACT == PCNN_ACT_RELU) yv[u] = ld<VEC>(y + off);
                    if (dy2) d2[u] = ld<VEC>(dy2 + off);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int px = p0 + lane + (j0 + u) * a.lanes;
                if (px >= a.HW) continue;
                BfVec<VEC> gv;
#pragma unroll
                for (int c = 0; c < VEC; ++c) {
                    gv.h[c] = se_dgrad<ACT>(dv[u].h[c], d2[u].h[c], dy2 != nullptr, yv[u].h[c]);
                    const float p = __fmul_rn(__bfloat162float(gv.h[c]), __bfloat162float(xv[u].h[c]));
                    acc[c] = j0 + u == 0 ? p : __fadd_rn(acc[c], p);
                }
                st<VEC>(g_out + base + (long)px * a.C, gv);
            }
        }
#pragma unroll
        for (int c = 0; c < VEC; ++c) part[lane * width + gl * VEC + c] = acc[c];
    }
    __syncthreads();
    const int active = min(a.lanes, a.HW - p0);            // lanes holding at least one pixel
    for (int t = threadIdx.x; t < width; t += SE_THREADS) {
        const int c = slice * width + t;
        if (c >= a.C) break;
        float sum = part[t];
        for (int l = 1; l < active; ++l) sum = __fadd_rn(sum, part[l * width + t]);
        if (a.ranges == 1)
            ds[(long)n * a.C + c] = __float2bfloat16_rn(sum);
        else
            slots[(long)nr * a.C + c] = sum;
    }
}

// one thread per (n, c): the slots of image n added in range order, ds = bf16_rn(sum)
__global__ void __launch_bounds__(SE_THREADS) k_se_finish(const float *__restrict__ slots, __nv_bfloat16 *__restrict__ ds, int N, GapArgs a) {
    const long i = (long)blockIdx.x * SE_THREADS + threadIdx.x;
    if (i >= (long)N * a.C) return;
    const int n = (int)(i / a.C), c = (int)(i - (long)n * a.C);
    const float *sl = slots + (long)n * a.ranges * a.C + c;
    float sum = sl[0];
    for (int r = 1; r < a.ranges; ++r) sum = __fadd_rn(sum, sl[(long)r * a.C]);
    ds[i] = __float2bfloat16_rn(sum);
}

// dx = bf16_rn(RN(float(g) * float(s)) (+ RN(float(dpool) / float(H W)), rounded once more by the add)).  dx may be g.
template <int VEC>
__global__ void __launch_bounds__(SE_THREADS) k_se_dx(const __nv_bfloat16 *g, const __nv_bfloat16 *__restrict__ s,
                                                      const __nv_bfloat16 *__restrict__ dpool, __nv_bfloat16 *dx, GapArgs a, int blocks) {
    const int n = blockIdx.x / blocks;
    const int i = (blockIdx.x - n * blocks) * SE_THREADS + threadIdx.x;
    if (i >= a.HW * a.G) return;
    const int gi = i % a.G;
    const long off = (long)n * a.HW * a.C + (long)i * VEC;
    const BfVec<VEC> gv = ld<VEC>(g + off);
    const BfVec<VEC> sv = ld<VEC>(s + (long)n * a.C + gi * VEC);
    BfVec<VEC> dp;
    if (dpool) dp = ld<VEC>(dpool + (long)n * a.pitch + gi * VEC);
    BfVec<VEC> out;
#pragma unroll
    for (int c = 0; c < VEC; ++c) {
        float v = __fmul_rn(__bfloat162float(gv.h[c]), __bfloat162float(sv.h[c]));
        if (dpool) v = __fadd_rn(v, div_rn(__bfloat162float(dp.h[c]), a.hw, a.rhw));
        out.h[c] = __float2bfloat16_rn(v);
    }
    st<VEC>(dx + off, out);
}

int se_act(const char *fn, int act) {
    PCNN_REQUIRE(act != PCNN_ACT_SIGMOID, PCNN_ERR_ARG,
                 "%s: act 1 (sigmoid) is not available after the channel scale: sigmoid_bf16 uses tanh.approx, which no reference "
                 "can replay bit for bit; act 0 (none) or 3 (ReLU) is required", fn);
    PCNN_REQUIRE(act == PCNN_ACT_NONE || act == PCNN_ACT_RELU, PCNN_ERR_ARG, "%s: act %d is not 0 (none) or 3 (ReLU)", fn, act);
    return PCNN_OK;
}

struct Buf {
    const void *p;
    size_t n;
};

bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// true when no two of the non-NULL buffers share a byte, except same_a and same_b when they are the same buffer (in place)
bool disjoint(const Buf *b, int n, const void *same_a, const void *same_b) {
    for (int i = 0; i < n; ++i)
        for (int j = i + 1; j < n; ++j) {
            if (!b[i].p || !b[j].p) continue;
            const uintptr_t pi = (uintptr_t)b[i].p, pj = (uintptr_t)b[j].p;
            if (!(pi < pj + b[j].n && pj < pi + b[i].n)) continue;
            const bool in_place = same_a && b[i].p == b[j].p && b[i].n == b[j].n &&
                                  ((b[i].p == same_a && b[j].p == same_b) || (b[i].p == same_b && b[j].p == same_a));
            if (!in_place) return false;
        }
    return true;
}

// CTAs per image of the elementwise passes (gap_shape has checked that N of them fit the grid)
int se_blocks(const GapArgs &a) { return (a.HW * a.G + SE_THREADS - 1) / SE_THREADS; }

typedef void (*fwd_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, __nv_bfloat16 *, GapArgs, int);
typedef void (*gate_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, __nv_bfloat16 *,
                        __nv_bfloat16 *, float *, GapArgs);

}  // namespace

extern "C" int pcnn_se_scale_nhwc_info(int N, int H, int W, int C, int *out8) {
    const char *fn = "pcnn_se_scale_nhwc_info";
    PCNN_REQUIRE(out8, PCNN_ERR_ARG, "%s: NULL out8", fn);
    GapArgs a;
    int rc = gap_shape(fn, N, H, W, C, 0, &a);
    if (rc) return rc;
    const int lane_pixels = std::min(GAP_ITERS, (a.HW + a.lanes - 1) / a.lanes), active = std::min(a.lanes, a.HW);
    out8[0] = C / a.G;
    out8[1] = a.Gc;
    out8[2] = a.slices;
    out8[3] = a.lanes;
    out8[4] = a.per_cta;
    out8[5] = a.ranges;
    out8[6] = N * a.ranges * a.slices;
    out8[7] = (lane_pixels - 1) + (active - 1) + (a.ranges - 1);
    return PCNN_OK;
}

extern "C" int pcnn_se_scale_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16, const void *s_bf16, const void *r_bf16, void *y_bf16, int N,
                                           int H, int W, int C, int act) {
    const char *fn = "pcnn_se_scale_nhwc_bf16_fwd";
    PCNN_REQUIRE(ctx && x_bf16 && s_bf16 && y_bf16, PCNN_ERR_ARG, "%s: NULL context, x, s or y (only r may be NULL)", fn);
    int rc = se_act(fn, act);
    if (rc) return rc;
    GapArgs a;
    if ((rc = gap_shape(fn, N, H, W, C, 0, &a))) return rc;
    PCNN_REQUIRE(aligned16(x_bf16) && aligned16(s_bf16) && aligned16(r_bf16) && aligned16(y_bf16), PCNN_ERR_ARG,
                 "%s: x, s, r and y must be 16-byte aligned", fn);
    const size_t tb = (size_t)N * a.HW * C * 2, sb = (size_t)N * C * 2;
    const Buf bufs[4] = {{x_bf16, tb}, {s_bf16, sb}, {r_bf16, tb}, {y_bf16, tb}};
    PCNN_REQUIRE(disjoint(bufs, 4, nullptr, nullptr), PCNN_ERR_ARG, "%s: overlapping buffers: x, s, r and y must not share memory", fn);
    pcnn_device_guard dg(ctx->device);
    const int blocks = se_blocks(a), v8 = C / a.G == 8 ? 1 : 0, relu = act == PCNN_ACT_RELU ? 1 : 0;
    static const fwd_fn table[2][2] = {{k_se_fwd<1, PCNN_ACT_NONE>, k_se_fwd<1, PCNN_ACT_RELU>},
                                       {k_se_fwd<8, PCNN_ACT_NONE>, k_se_fwd<8, PCNN_ACT_RELU>}};
    table[v8][relu]<<<(unsigned)((long)N * blocks), SE_THREADS, 0, ctx->stream>>>(
        static_cast<const __nv_bfloat16 *>(x_bf16), static_cast<const __nv_bfloat16 *>(s_bf16), static_cast<const __nv_bfloat16 *>(r_bf16),
        static_cast<__nv_bfloat16 *>(y_bf16), a, blocks);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_se_scale_nhwc_bf16_bwd_gate(pcnn_ctx *ctx, const void *x_bf16, const void *y_bf16, const void *dy_bf16,
                                                const void *dy2_bf16, void *g_bf16, void *ds_bf16, int N, int H, int W, int C, int act) {
    const char *fn = "pcnn_se_scale_nhwc_bf16_bwd_gate";
    PCNN_REQUIRE(ctx && x_bf16 && dy_bf16 && g_bf16 && ds_bf16, PCNN_ERR_ARG,
                 "%s: NULL context, x, dy, g or ds (only y at act 0 and dy2 may be NULL)", fn);
    int rc = se_act(fn, act);
    if (rc) return rc;
    PCNN_REQUIRE(act != PCNN_ACT_RELU || y_bf16, PCNN_ERR_ARG, "%s: act 3 (ReLU) needs y, the forward's output (NULL given)", fn);
    GapArgs a;
    if ((rc = gap_shape(fn, N, H, W, C, 0, &a))) return rc;
    const void *ptrs[6] = {x_bf16, y_bf16, dy_bf16, dy2_bf16, g_bf16, ds_bf16};
    for (const void *q : ptrs) PCNN_REQUIRE(aligned16(q), PCNN_ERR_ARG, "%s: x, y, dy, dy2, g and ds must be 16-byte aligned", fn);
    const size_t tb = (size_t)N * a.HW * C * 2, sb = (size_t)N * C * 2;
    const Buf bufs[6] = {{x_bf16, tb}, {y_bf16, tb}, {dy_bf16, tb}, {dy2_bf16, tb}, {g_bf16, tb}, {ds_bf16, sb}};
    PCNN_REQUIRE(disjoint(bufs, 6, g_bf16, dy_bf16), PCNN_ERR_ARG, "%s: overlapping buffers: only g == dy (in place) may share memory", fn);
    pcnn_device_guard dg(ctx->device);
    float *slots = nullptr;
    if (a.ranges > 1 && (rc = pcnn_scratch(ctx, (size_t)N * a.ranges * C * sizeof(float), (void **)&slots))) return rc;
    const int v8 = C / a.G == 8 ? 1 : 0, relu = act == PCNN_ACT_RELU ? 1 : 0;
    static const gate_fn table[2][2] = {{k_se_gate<1, PCNN_ACT_NONE>, k_se_gate<1, PCNN_ACT_RELU>},
                                        {k_se_gate<8, PCNN_ACT_NONE>, k_se_gate<8, PCNN_ACT_RELU>}};
    auto *ds = static_cast<__nv_bfloat16 *>(ds_bf16);
    table[v8][relu]<<<(unsigned)((long)N * a.ranges * a.slices), SE_THREADS, 0, ctx->stream>>>(
        static_cast<const __nv_bfloat16 *>(x_bf16), static_cast<const __nv_bfloat16 *>(y_bf16), static_cast<const __nv_bfloat16 *>(dy_bf16),
        static_cast<const __nv_bfloat16 *>(dy2_bf16), static_cast<__nv_bfloat16 *>(g_bf16), ds, slots, a);
    PCNN_CHECK_LAUNCH(ctx);
    if (a.ranges > 1) {
        k_se_finish<<<(unsigned)(((long)N * C + SE_THREADS - 1) / SE_THREADS), SE_THREADS, 0, ctx->stream>>>(slots, ds, N, a);
        PCNN_CHECK_LAUNCH(ctx);
    }
    return PCNN_OK;
}

extern "C" int pcnn_se_scale_nhwc_bf16_bwd_input(pcnn_ctx *ctx, const void *g_bf16, const void *s_bf16, const void *dpool_bf16,
                                                 int dpool_row_pitch, void *dx_bf16, int N, int H, int W, int C) {
    const char *fn = "pcnn_se_scale_nhwc_bf16_bwd_input";
    PCNN_REQUIRE(ctx && g_bf16 && s_bf16 && dx_bf16, PCNN_ERR_ARG, "%s: NULL context, g, s or dx (only dpool may be NULL)", fn);
    GapArgs a;
    int rc = gap_shape(fn, N, H, W, C, dpool_row_pitch, &a);
    if (rc) return rc;
    PCNN_REQUIRE(aligned16(g_bf16) && aligned16(s_bf16) && aligned16(dpool_bf16) && aligned16(dx_bf16), PCNN_ERR_ARG,
                 "%s: g, s, dpool and dx must be 16-byte aligned", fn);
    const size_t tb = (size_t)N * a.HW * C * 2, sb = (size_t)N * C * 2, pb = (size_t)N * a.pitch * 2;
    const Buf bufs[4] = {{g_bf16, tb}, {s_bf16, sb}, {dpool_bf16, pb}, {dx_bf16, tb}};
    PCNN_REQUIRE(disjoint(bufs, 4, dx_bf16, g_bf16), PCNN_ERR_ARG, "%s: overlapping buffers: only dx == g (in place) may share memory", fn);
    pcnn_device_guard dg(ctx->device);
    const int blocks = se_blocks(a);
    const unsigned grid = (unsigned)((long)N * blocks);
    const auto *g = static_cast<const __nv_bfloat16 *>(g_bf16);
    const auto *s = static_cast<const __nv_bfloat16 *>(s_bf16);
    const auto *dpool = static_cast<const __nv_bfloat16 *>(dpool_bf16);
    auto *dx = static_cast<__nv_bfloat16 *>(dx_bf16);
    if (C / a.G == 8)
        k_se_dx<8><<<grid, SE_THREADS, 0, ctx->stream>>>(g, s, dpool, dx, a, blocks);
    else
        k_se_dx<1><<<grid, SE_THREADS, 0, ctx->stream>>>(g, s, dpool, dx, a, blocks);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
