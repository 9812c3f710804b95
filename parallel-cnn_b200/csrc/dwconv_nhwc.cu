// parallel-cnn_b200/csrc/dwconv_nhwc.cu -- depthwise convolution (groups = C: each channel filtered by its own R x S filter)
// between bf16 NHWC layers: pcnn_dwconv_plan_create (a pcnn_conv_plan run by pcnn_conv_tc_fwd, refreshed by
// pcnn_conv_plan_set_params and the optimizer), pcnn_dwconv_wgrad, pcnn_dwconv_dgrad and pcnn_dwconv_info.  The contract is in
// include/pcnn.h.
//
// All three passes are HBM-bound (about 2 R S flops per 4 bytes moved).  With C % 8 == 0 a thread moves 16-byte vectors of 8
// channels of one pixel, otherwise single elements.  A CTA owns a slice of at most DW_MAX_GROUPS channel groups and stages their
// bf16 filters, [C][R][S] in the plan, through shared memory as [tap][channel].
//   - Forward: thread (strip, group) computes DW_QS consecutive outputs along q of one output row; at stride < S neighbouring
//     outputs share x columns, so each x column of the strip is loaded once per filter row.
//   - Input gradient: a gather like the pool backward.  Thread (strip, group) owns DW_QS consecutive dx elements along w; it visits
//     the dy rows on the stride grid in ascending r and, within a row, the dy columns in descending q (ascending s), so every dx
//     element sums its terms in the order pcnn.h states and is written once, with no memset and no atomics.
//   - Weight gradient: CTA (pixel range, channel slice) walks filter rows r; each thread keeps S x VEC fp32 sums of one filter row
//     over the pixels lane, lane + lanes, ... of its range, the lanes are added in lane order through shared memory, and each range
//     writes an fp32 slot [C][R][S] that pcnn_conv_wgrad_reduce_slots adds in a fixed order.  The ranges depend on the shape only.
// Dilation (pcnn_dwconv_plan_create_dilated): tap (r, s) sits r*dil_h rows and s*dil_w columns from the window's corner.  Each pass
// has a second instantiation (DIL), so the undilated ones keep their code.  The DIL forward walks the taps of each output (for r, s,
// output k: x column q0 st + k st + s dil_w, repeats served by L1), so it loads no column that no output of the strip reads; the DIL
// input gradient walks each element's taps in ascending s and finds the dy column (w + pad_w - s dil_w) / stride; the DIL weight
// gradient reads x at w0 + s*dil_w.  The orders stay those stated above.
#include "pcnn_internal.h"

#include <cuda_bf16.h>

#include <memory>

namespace {

constexpr int DW_THREADS = 256;
constexpr int DW_MAX_TAPS = 7;
constexpr int DW_MAX_GROUPS = 32;          // channel groups per CTA: 256 channels on the 16-byte path
constexpr int DW_QS = 4;                   // outputs (forward) or dx elements (input gradient) per thread along a row
constexpr int DW_ITERS = 16;               // pixels per thread of the weight gradient

template <int VEC>
struct alignas(2 * VEC) BfVec {
    __nv_bfloat16 h[VEC];
};

struct DwArgs {
    int N, H, W, C, R, S, stride, pad_h, pad_w, P, Q;
    int G;                  // channel groups of VEC channels
    int Gc, slices;         // groups per CTA, channel slices (the last may hold fewer groups)
    int lanes;              // 256 / Gc: strips (forward, input gradient) or pixel lanes (weight gradient) per CTA
    int qb, wb;             // strips per output row (forward) and per input row (input gradient)
    long long fstrips, dstrips;   // N P qb, N H wb
    long long M;            // N P Q output pixels
    int per_range, ranges;  // weight gradient: pixels per range (lanes * DW_ITERS) and ranges
    int act;
    int dil_h, dil_w;       // dilation (1 = none)
};

template <int VEC>
__device__ __forceinline__ BfVec<VEC> bf_zero() {
    BfVec<VEC> v;
#pragma unroll
    for (int c = 0; c < VEC; ++c) v.h[c] = __ushort_as_bfloat16(0);
    return v;
}

// the slice's bf16 filters [C][R][S] -> shared [tap][Gc * VEC]
__device__ __forceinline__ void stage_filters(const __nv_bfloat16 *__restrict__ wop, __nv_bfloat16 *wsm, const DwArgs &a, int c0, int cs,
                                              int stride_sm) {
    const int RS = a.R * a.S;
    for (int i = threadIdx.x; i < cs * RS; i += DW_THREADS) {
        const int c = i / RS, t = i - c * RS;
        wsm[t * stride_sm + c] = wop[(long)(c0 + c) * RS + t];
    }
}

template <int VEC, bool DIL>
__global__ void __launch_bounds__(DW_THREADS) k_dwconv_fwd(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ wop,
                                                           const float *__restrict__ bias, __nv_bfloat16 *__restrict__ y, DwArgs a) {
    __shared__ __align__(16) __nv_bfloat16 wsm[DW_MAX_TAPS * DW_MAX_TAPS * DW_MAX_GROUPS * VEC];
    const int width = a.Gc * VEC, c0 = blockIdx.y * width, cs = min(width, a.C - c0);
    stage_filters(wop, wsm, a, c0, cs, width);
    __syncthreads();
    const int gl = threadIdx.x % a.Gc, lane = threadIdx.x / a.Gc;
    const long long strip = (long long)blockIdx.x * a.lanes + lane;
    if (lane >= a.lanes || gl * VEC >= cs || strip >= a.fstrips) return;
    const int n = (int)(strip / ((long long)a.P * a.qb));
    const int rem = (int)(strip - (long long)n * a.P * a.qb), p = rem / a.qb, q0 = (rem - p * a.qb) * DW_QS;
    const int c = c0 + gl * VEC, st = a.stride;
    const __nv_bfloat16 *xi = x + (long)n * a.H * a.W * a.C + c;
    const __nv_bfloat16 *wg = wsm + gl * VEC;
    float acc[DW_QS][VEC];                                 // -0 + t == t for every t: each sum starts from its first term
#pragma unroll
    for (int k = 0; k < DW_QS; ++k)
#pragma unroll
        for (int e = 0; e < VEC; ++e) acc[k][e] = -0.0f;
    const int ncols = (DW_QS - 1) * st + a.S, wstart = q0 * st - a.pad_w;
    for (int r = 0; r < a.R; ++r) {
        const int h = p * st - a.pad_h + r * (DIL ? a.dil_h : 1);
        const bool rowok = h >= 0 && h < a.H;
        const __nv_bfloat16 *row = xi + (long)h * a.W * a.C;
        if (DIL) {                                         // tap by tap: only the columns some output of the strip reads
            for (int s = 0; s < a.S; ++s) {
                const BfVec<VEC> wv = *reinterpret_cast<const BfVec<VEC> *>(wg + (r * a.S + s) * width);
#pragma unroll
                for (int k = 0; k < DW_QS; ++k) {
                    const int w = wstart + k * st + s * a.dil_w;
                    if (q0 + k >= a.Q) continue;
                    BfVec<VEC> xv = bf_zero<VEC>();
                    if (rowok && w >= 0 && w < a.W) xv = *reinterpret_cast<const BfVec<VEC> *>(row + (long)w * a.C);
#pragma unroll
                    for (int e = 0; e < VEC; ++e) acc[k][e] = fmaf(__bfloat162float(xv.h[e]), __bfloat162float(wv.h[e]), acc[k][e]);
                }
            }
            continue;
        }
        for (int j = 0; j < ncols; ++j) {
            const int w = wstart + j;
            BfVec<VEC> xv = bf_zero<VEC>();
            if (rowok && w >= 0 && w < a.W) xv = *reinterpret_cast<const BfVec<VEC> *>(row + (long)w * a.C);
#pragma unroll
            for (int k = 0; k < DW_QS; ++k) {
                const int s = j - k * st;
                if (s < 0 || s >= a.S || q0 + k >= a.Q) continue;
                const BfVec<VEC> wv = *reinterpret_cast<const BfVec<VEC> *>(wg + (r * a.S + s) * width);
#pragma unroll
                for (int e = 0; e < VEC; ++e) acc[k][e] = fmaf(__bfloat162float(xv.h[e]), __bfloat162float(wv.h[e]), acc[k][e]);
            }
        }
    }
    __nv_bfloat16 *yo = y + (((long)n * a.P + p) * a.Q + q0) * a.C + c;
#pragma unroll
    for (int k = 0; k < DW_QS; ++k) {
        if (q0 + k >= a.Q) break;
        BfVec<VEC> out;
#pragma unroll
        for (int e = 0; e < VEC; ++e) {
            float v = bias ? __fadd_rn(acc[k][e], bias[c + e]) : acc[k][e];
            if (a.act == PCNN_ACT_RELU) v = v < 0.0f ? 0.0f : v;
            out.h[e] = __float2bfloat16_rn(v);
        }
        *reinterpret_cast<BfVec<VEC> *>(yo + (long)k * a.C) = out;
    }
}

template <int VEC, bool DIL>
__global__ void __launch_bounds__(DW_THREADS) k_dwconv_dgrad(const __nv_bfloat16 *__restrict__ dy, const __nv_bfloat16 *__restrict__ wop,
                                                             __nv_bfloat16 *__restrict__ dx, DwArgs a) {
    __shared__ __align__(16) __nv_bfloat16 wsm[DW_MAX_TAPS * DW_MAX_TAPS * DW_MAX_GROUPS * VEC];
    const int width = a.Gc * VEC, c0 = blockIdx.y * width, cs = min(width, a.C - c0);
    stage_filters(wop, wsm, a, c0, cs, width);
    __syncthreads();
    const int gl = threadIdx.x % a.Gc, lane = threadIdx.x / a.Gc;
    const long long strip = (long long)blockIdx.x * a.lanes + lane;
    if (lane >= a.lanes || gl * VEC >= cs || strip >= a.dstrips) return;
    const int n = (int)(strip / ((long long)a.H * a.wb));
    const int rem = (int)(strip - (long long)n * a.H * a.wb), h = rem / a.wb, w0 = (rem - h * a.wb) * DW_QS;
    const int c = c0 + gl * VEC, st = a.stride;
    const __nv_bfloat16 *dyi = dy + (long)n * a.P * a.Q * a.C + c;
    const __nv_bfloat16 *wg = wsm + gl * VEC;
    float acc[DW_QS][VEC];
#pragma unroll
    for (int k = 0; k < DW_QS; ++k)
#pragma unroll
        for (int e = 0; e < VEC; ++e) acc[k][e] = -0.0f;
    bool khit[DW_QS] = {};                                 // DIL: element k has a term
    // dy columns q with 0 <= w + pad_w - q stride < S for some w of the strip, inside [0, Q)
    const int nw = w0 + a.pad_w - a.S + 1;
    const int qlo = nw <= 0 ? 0 : (nw + st - 1) / st, qhi = min(a.Q - 1, (w0 + DW_QS - 1 + a.pad_w) / st);
    bool rowhit = false;
    for (int r = 0; r < a.R; ++r) {
        const int t = h + a.pad_h - r * (DIL ? a.dil_h : 1);
        if (t < 0 || t % st != 0 || t / st >= a.P) continue;
        rowhit = true;
        const __nv_bfloat16 *row = dyi + (long)(t / st) * a.Q * a.C;
        if (DIL) {                                         // element by element, taps in ascending s: only the dy columns read
#pragma unroll
            for (int k = 0; k < DW_QS; ++k) {
                for (int s = 0; s < a.S; ++s) {
                    const int u = w0 + k + a.pad_w - s * a.dil_w;
                    if (u < 0) break;
                    if (u % st != 0 || u / st >= a.Q) continue;
                    khit[k] = true;
                    const BfVec<VEC> d = *reinterpret_cast<const BfVec<VEC> *>(row + (long)(u / st) * a.C);
                    const BfVec<VEC> wv = *reinterpret_cast<const BfVec<VEC> *>(wg + (r * a.S + s) * width);
#pragma unroll
                    for (int e = 0; e < VEC; ++e) acc[k][e] = fmaf(__bfloat162float(d.h[e]), __bfloat162float(wv.h[e]), acc[k][e]);
                }
            }
            continue;
        }
        for (int q = qhi; q >= qlo; --q) {                 // descending q: ascending s for every element of the strip
            const BfVec<VEC> d = *reinterpret_cast<const BfVec<VEC> *>(row + (long)q * a.C);
#pragma unroll
            for (int k = 0; k < DW_QS; ++k) {
                const int s = w0 + k + a.pad_w - q * st;
                if (s < 0 || s >= a.S) continue;
                const BfVec<VEC> wv = *reinterpret_cast<const BfVec<VEC> *>(wg + (r * a.S + s) * width);
#pragma unroll
                for (int e = 0; e < VEC; ++e) acc[k][e] = fmaf(__bfloat162float(d.h[e]), __bfloat162float(wv.h[e]), acc[k][e]);
            }
        }
    }
    __nv_bfloat16 *dxo = dx + (((long)n * a.H + h) * a.W + w0) * a.C + c;
#pragma unroll
    for (int k = 0; k < DW_QS; ++k) {
        const int w = w0 + k;
        if (w >= a.W) break;
        // the taps of (h, w) are the valid rows times the valid columns: none when either set is empty
        const int nk = w + a.pad_w - a.S + 1;
        const int ql = nk <= 0 ? 0 : (nk + st - 1) / st, qh = min(a.Q - 1, (w + a.pad_w) / st);
        const bool hit = DIL ? khit[k] : rowhit && ql <= qh;
        BfVec<VEC> out;
#pragma unroll
        for (int e = 0; e < VEC; ++e) out.h[e] = hit ? __float2bfloat16_rn(acc[k][e]) : __ushort_as_bfloat16(0);
        *reinterpret_cast<BfVec<VEC> *>(dxo + (long)k * a.C) = out;
    }
}

// CTA (range, slice): out[c][r][s] for the slice's channels over the pixels [range * per_range, (range + 1) * per_range) of the
// N P Q output pixels; `out` is dw itself when there is one range, otherwise slot `range` of the [ranges][C][R][S] partials
template <int VEC, int S, bool DIL>
__global__ void __launch_bounds__(DW_THREADS) k_dwconv_wgrad(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ dy,
                                                             float *__restrict__ out, DwArgs a) {
    __shared__ float part[DW_THREADS * 8];                 // [lanes][Gc * VEC]
    const int width = a.Gc * VEC, c0 = blockIdx.y * width, cs = min(width, a.C - c0);
    const int gl = threadIdx.x % a.Gc, lane = threadIdx.x / a.Gc, c = c0 + gl * VEC;
    const bool on = lane < a.lanes && gl * VEC < cs;
    const long long p0 = (long long)blockIdx.x * a.per_range;
    const int active = (int)min((long long)a.lanes, a.M - p0);   // lanes holding at least one pixel
    const int st = a.stride, PQ = a.P * a.Q;
    float *slot = out + (long)blockIdx.x * a.C * a.R * S;
    for (int r = 0; r < a.R; ++r) {
        float acc[S][VEC];
#pragma unroll
        for (int s = 0; s < S; ++s)
#pragma unroll
            for (int e = 0; e < VEC; ++e) acc[s][e] = -0.0f;
        if (on) {
            for (int i = 0; i < DW_ITERS; ++i) {
                const long long m = p0 + lane + (long long)i * a.lanes;
                if (m >= a.M || m >= p0 + a.per_range) break;
                const int n = (int)(m / PQ), pq = (int)(m - (long long)n * PQ), p = pq / a.Q, q = pq - p * a.Q;
                const BfVec<VEC> d = *reinterpret_cast<const BfVec<VEC> *>(dy + m * a.C + c);
                const int h = p * st - a.pad_h + r * (DIL ? a.dil_h : 1), w0 = q * st - a.pad_w;
                const bool rowok = h >= 0 && h < a.H;
                const __nv_bfloat16 *row = x + ((long)n * a.H + h) * a.W * a.C + c;
#pragma unroll
                for (int s = 0; s < S; ++s) {
                    const int w = w0 + s * (DIL ? a.dil_w : 1);
                    BfVec<VEC> xv = bf_zero<VEC>();
                    if (rowok && w >= 0 && w < a.W) xv = *reinterpret_cast<const BfVec<VEC> *>(row + (long)w * a.C);
#pragma unroll
                    for (int e = 0; e < VEC; ++e) acc[s][e] = fmaf(__bfloat162float(d.h[e]), __bfloat162float(xv.h[e]), acc[s][e]);
                }
            }
        }
#pragma unroll
        for (int s = 0; s < S; ++s) {
            if (on)
#pragma unroll
                for (int e = 0; e < VEC; ++e) part[lane * width + gl * VEC + e] = acc[s][e];
            __syncthreads();
            for (int t = threadIdx.x; t < cs; t += DW_THREADS) {
                float v = part[t];
                for (int l = 1; l < active; ++l) v = __fadd_rn(v, part[l * width + t]);
                slot[((long)(c0 + t) * a.R + r) * S + s] = v;
            }
            __syncthreads();
        }
    }
}

}  // namespace

namespace {

constexpr int DW_MAX_DIL = 256;

// nhwc_window_check with a dilation: at (1, 1) exactly it, messages included
int nhwc_window_check_dilated(const char *fn, int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int dil_h,
                              int dil_w, int *P, int *Q) {
    PCNN_REQUIRE(N >= 1 && H >= 1 && W >= 1 && C >= 1, PCNN_ERR_ARG, "%s: N = %d, H = %d, W = %d, C = %d: each must be >= 1", fn, N, H, W,
                 C);
    PCNN_REQUIRE(R >= 1 && R <= DW_MAX_TAPS && S >= 1 && S <= DW_MAX_TAPS, PCNN_ERR_ARG, "%s: %dx%d filter: 1 <= R, S <= 7 is required",
                 fn, R, S);
    PCNN_REQUIRE(stride >= 1 && stride <= 4, PCNN_ERR_ARG, "%s: stride %d: 1 <= stride <= 4 is required", fn, stride);
    PCNN_REQUIRE(dil_h >= 1 && dil_h <= DW_MAX_DIL && dil_w >= 1 && dil_w <= DW_MAX_DIL, PCNN_ERR_ARG,
                 "%s: dilation (%d, %d): 1 <= dil_h, dil_w <= %d are required", fn, dil_h, dil_w, DW_MAX_DIL);
    const int Eh = dil_h * (R - 1) + 1, Ew = dil_w * (S - 1) + 1;     // the window's extent
    if (dil_h == 1 && dil_w == 1) {
        PCNN_REQUIRE(pad_h >= 0 && pad_h <= R - 1 && pad_w >= 0 && pad_w <= S - 1, PCNN_ERR_ARG,
                     "%s: padding (%d, %d) for a %dx%d filter: 0 <= pad_h <= R - 1 and 0 <= pad_w <= S - 1 are required", fn, pad_h, pad_w,
                     R, S);
        PCNN_REQUIRE(H + 2 * pad_h >= R && W + 2 * pad_w >= S, PCNN_ERR_ARG,
                     "%s: a %dx%d filter does not fit the %dx%d image padded by (%d, %d): H + 2 pad_h >= R and W + 2 pad_w >= S are required",
                     fn, R, S, H, W, pad_h, pad_w);
    } else {
        PCNN_REQUIRE(pad_h >= 0 && pad_h <= Eh - 1 && pad_w >= 0 && pad_w <= Ew - 1, PCNN_ERR_ARG,
                     "%s: padding (%d, %d) for a %dx%d filter at dilation (%d, %d): 0 <= pad_h <= dil_h (R - 1) and 0 <= pad_w <= dil_w (S - 1) "
                     "are required", fn, pad_h, pad_w, R, S, dil_h, dil_w);
        PCNN_REQUIRE(H + 2 * pad_h >= Eh && W + 2 * pad_w >= Ew, PCNN_ERR_ARG,
                     "%s: a %dx%d filter at dilation (%d, %d) does not fit the %dx%d image padded by (%d, %d): H + 2 pad_h >= dil_h (R - 1) + 1 "
                     "and W + 2 pad_w >= dil_w (S - 1) + 1 are required", fn, R, S, dil_h, dil_w, H, W, pad_h, pad_w);
    }
    *P = (H + 2 * pad_h - Eh) / stride + 1;
    *Q = (W + 2 * pad_w - Ew) / stride + 1;
    return PCNN_OK;
}

}  // namespace

int nhwc_window_check(const char *fn, int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int *P, int *Q) {
    return nhwc_window_check_dilated(fn, N, H, W, C, R, S, stride, pad_h, pad_w, 1, 1, P, Q);
}

namespace {

// the domain of pcnn.h, refused with PCNN_ERR_ARG and a message naming `fn`, and the partition, a function of the shape alone
int dw_shape(const char *fn, int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int dil_h, int dil_w, DwArgs *a) {
    int P, Q;
    const int rc = nhwc_window_check_dilated(fn, N, H, W, C, R, S, stride, pad_h, pad_w, dil_h, dil_w, &P, &Q);
    if (rc) return rc;
    PCNN_REQUIRE((long)H * W * C <= INT32_MAX && (long)P * Q * C <= INT32_MAX && (long)C * R * S <= INT32_MAX, PCNN_ERR_ARG,
                 "%s: one %dx%dx%d image (or its %d x %d x %d filters) exceeds the 32-bit index range: H W C, P Q C and C R S < 2^31 are "
                 "required", fn, H, W, C, C, R, S);
    const int vec = C % 8 == 0 ? 8 : 1, G = C / vec;
    a->N = N; a->H = H; a->W = W; a->C = C; a->R = R; a->S = S; a->stride = stride; a->pad_h = pad_h; a->pad_w = pad_w; a->P = P; a->Q = Q;
    a->G = G;
    a->slices = (G + DW_MAX_GROUPS - 1) / DW_MAX_GROUPS;
    a->Gc = (G + a->slices - 1) / a->slices;
    a->lanes = DW_THREADS / a->Gc;
    a->qb = (Q + DW_QS - 1) / DW_QS;
    a->wb = (W + DW_QS - 1) / DW_QS;
    a->fstrips = (long long)N * P * a->qb;
    a->dstrips = (long long)N * H * a->wb;
    a->M = (long long)N * P * Q;
    a->per_range = a->lanes * DW_ITERS;
    const long long ranges = (a->M + a->per_range - 1) / a->per_range;
    PCNN_REQUIRE(a->slices <= 65535 && ranges <= INT32_MAX && (a->fstrips + a->lanes - 1) / a->lanes <= INT32_MAX &&
                     (a->dstrips + a->lanes - 1) / a->lanes <= INT32_MAX,
                 PCNN_ERR_ARG, "%s: %d images of %dx%dx%d exceed the grid", fn, N, H, W, C);
    a->ranges = (int)ranges;
    a->act = 0;
    a->dil_h = dil_h; a->dil_w = dil_w;
    return PCNN_OK;
}

// additions on the longest path of one weight-gradient sum: the pixels of a lane, the lanes of a range, then (with several
// ranges) pcnn_conv_wgrad_reduce_slots: every 8th slot added to +0, then a tree over the 8
int dw_n_acc(const DwArgs &a) {
    const int lane_px = a.M < a.per_range ? (int)((a.M + a.lanes - 1) / a.lanes) : DW_ITERS;
    const int lanes = (int)(a.M < a.lanes ? a.M : a.lanes);
    return (lane_px - 1) + (lanes - 1) + (a.ranges > 1 ? (a.ranges + 7) / 8 + 3 : 0);
}

bool overlap(const void *p, size_t np, const void *q, size_t nq) {
    const uintptr_t a = (uintptr_t)p, b = (uintptr_t)q;
    return a < b + nq && b < a + np;
}

bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

typedef void (*wgrad_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, float *, DwArgs);
template <int VEC, bool DIL>
wgrad_fn wgrad_variant(int S) {
    static const wgrad_fn t[DW_MAX_TAPS] = {k_dwconv_wgrad<VEC, 1, DIL>, k_dwconv_wgrad<VEC, 2, DIL>, k_dwconv_wgrad<VEC, 3, DIL>,
                                            k_dwconv_wgrad<VEC, 4, DIL>, k_dwconv_wgrad<VEC, 5, DIL>, k_dwconv_wgrad<VEC, 6, DIL>,
                                            k_dwconv_wgrad<VEC, 7, DIL>};
    return t[S - 1];
}

}  // namespace

// a plan of pcnn_dwconv_plan_create(_dilated): w is [C][R][S], the fp32 master's element order (one row of n elements)
struct DwConvPlan : pcnn_conv_plan {
    static constexpr const char *made_by = "pcnn_dwconv_plan_create";
    DwArgs a;
    const __nv_bfloat16 *wop() const { return static_cast<const __nv_bfloat16 *>(w); }
    int fwd(pcnn_ctx *ctx, const void *x_bf16, void *y_bf16) override;
};

static int dw_info(const char *fn, int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int dil_h, int dil_w,
                   int *out9) {
    PCNN_REQUIRE(out9, PCNN_ERR_ARG, "%s: NULL out9", fn);
    DwArgs a;
    int rc = dw_shape(fn, N, H, W, C, R, S, stride, pad_h, pad_w, dil_h, dil_w, &a);
    if (rc) return rc;
    const int v[9] = {a.P, a.Q, C % 8 == 0 ? 8 : 1, a.Gc, a.slices, a.lanes, a.per_range, a.ranges, dw_n_acc(a)};
    memcpy(out9, v, sizeof(v));
    return PCNN_OK;
}

extern "C" int pcnn_dwconv_info(int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int *out9) {
    return dw_info("pcnn_dwconv_info", N, H, W, C, R, S, stride, pad_h, pad_w, 1, 1, out9);
}

extern "C" int pcnn_dwconv_info_dilated(int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int dil_h, int dil_w,
                                        int *out9) {
    return dw_info("pcnn_dwconv_info_dilated", N, H, W, C, R, S, stride, pad_h, pad_w, dil_h, dil_w, out9);
}

static int dw_plan_create(const char *fn, pcnn_ctx *ctx, int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w,
                          int dil_h, int dil_w, int act, const float *filt_host, const float *bias_host, pcnn_conv_plan **out) {
    PCNN_REQUIRE(ctx && filt_host && out, PCNN_ERR_ARG, "%s: NULL context, filters or out", fn);
    PCNN_REQUIRE_ACT(fn, act);
    PCNN_REQUIRE(act != PCNN_ACT_SIGMOID, PCNN_ERR_ARG,
                 "%s: act 1 (sigmoid) is not supported: the sigmoid of the conv epilogues uses tanh.approx, which no reference can replay "
                 "bit for bit; use act 0 or 3", fn);
    DwArgs a;
    int rc = dw_shape(fn, N, H, W, C, R, S, stride, pad_h, pad_w, dil_h, dil_w, &a);
    if (rc) return rc;
    a.act = act;
    pcnn_device_guard g(ctx->device);
    std::unique_ptr<DwConvPlan> pl(new DwConvPlan());   // frees a half-built plan on every early return below
    pl->a = a;
    pl->n = (long long)C * R * S;
    pl->cols = pl->pitch = (int)pl->n;
    pl->K = C;
    if ((rc = pcnn_plan_upload(ctx, pl.get(), &pl->w, (size_t)pl->n * 2, filt_host, bias_host))) return rc;
    *out = pl.release();
    return PCNN_OK;
}

extern "C" int pcnn_dwconv_plan_create(pcnn_ctx *ctx, int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int act,
                                       const float *filt_host, const float *bias_host, pcnn_conv_plan **out) {
    return dw_plan_create("pcnn_dwconv_plan_create", ctx, N, H, W, C, R, S, stride, pad_h, pad_w, 1, 1, act, filt_host, bias_host, out);
}

extern "C" int pcnn_dwconv_plan_create_dilated(pcnn_ctx *ctx, int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w,
                                               int dil_h, int dil_w, int act, const float *filt_host, const float *bias_host,
                                               pcnn_conv_plan **out) {
    return dw_plan_create("pcnn_dwconv_plan_create_dilated", ctx, N, H, W, C, R, S, stride, pad_h, pad_w, dil_h, dil_w, act, filt_host,
                          bias_host, out);
}

int DwConvPlan::fwd(pcnn_ctx *ctx, const void *x_bf16, void *y_bf16) {
    const char *fn = "pcnn_conv_tc_fwd";
    PCNN_REQUIRE(aligned16(y_bf16), PCNN_ERR_ARG, "%s: the output must be 16-byte aligned", fn);
    const size_t xb = (size_t)a.N * a.H * a.W * a.C * 2, yb = (size_t)a.M * a.C * 2;
    PCNN_REQUIRE(!overlap(x_bf16, xb, y_bf16, yb), PCNN_ERR_ARG, "%s: overlapping buffers: x and y of a depthwise plan must not share memory",
                 fn);
    const dim3 grid((unsigned)((a.fstrips + a.lanes - 1) / a.lanes), (unsigned)a.slices);
    const auto *x = static_cast<const __nv_bfloat16 *>(x_bf16);
    auto *y = static_cast<__nv_bfloat16 *>(y_bf16);
    const bool dil = a.dil_h > 1 || a.dil_w > 1;
    if (a.C % 8 == 0)
        (dil ? k_dwconv_fwd<8, true> : k_dwconv_fwd<8, false>)<<<grid, DW_THREADS, 0, ctx->stream>>>(x, wop(), bias, y, a);
    else
        (dil ? k_dwconv_fwd<1, true> : k_dwconv_fwd<1, false>)<<<grid, DW_THREADS, 0, ctx->stream>>>(x, wop(), bias, y, a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_dwconv_wgrad(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *x_bf16, const void *dy_bf16, float *dw_f32) {
    const char *fn = "pcnn_dwconv_wgrad";
    PCNN_REQUIRE(ctx && plan && x_bf16 && dy_bf16 && dw_f32, PCNN_ERR_ARG, "%s: NULL argument", fn);
    DwConvPlan *pl;
    int rc = plan_as(fn, plan, &pl);
    if (rc) return rc;
    PCNN_REQUIRE(aligned16(x_bf16) && aligned16(dy_bf16) && aligned16(dw_f32), PCNN_ERR_ARG, "%s: x, dy and dw must be 16-byte aligned", fn);
    const DwArgs &a = pl->a;
    const size_t xb = (size_t)a.N * a.H * a.W * a.C * 2, yb = (size_t)a.M * a.C * 2, nout = (size_t)a.C * a.R * a.S;
    PCNN_REQUIRE(!overlap(dw_f32, nout * 4, x_bf16, xb) && !overlap(dw_f32, nout * 4, dy_bf16, yb), PCNN_ERR_ARG,
                 "%s: overlapping buffers: dw must not share memory with x or dy", fn);
    pcnn_device_guard g(ctx->device);
    float *out = dw_f32;
    if (a.ranges > 1 && (rc = pcnn_scratch(ctx, (size_t)a.ranges * nout * sizeof(float), (void **)&out))) return rc;
    const dim3 grid((unsigned)a.ranges, (unsigned)a.slices);
    const auto *x = static_cast<const __nv_bfloat16 *>(x_bf16);
    const auto *dy = static_cast<const __nv_bfloat16 *>(dy_bf16);
    const bool dil = a.dil_h > 1 || a.dil_w > 1;
    const wgrad_fn k = a.C % 8 == 0 ? (dil ? wgrad_variant<8, true>(a.S) : wgrad_variant<8, false>(a.S))
                                    : (dil ? wgrad_variant<1, true>(a.S) : wgrad_variant<1, false>(a.S));
    k<<<grid, DW_THREADS, 0, ctx->stream>>>(x, dy, out, a);
    PCNN_CHECK_LAUNCH(ctx);
    return a.ranges > 1 ? pcnn_conv_wgrad_reduce_slots(ctx, out, dw_f32, a.ranges, (int)nout) : PCNN_OK;
}

extern "C" int pcnn_dwconv_dgrad(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *dy_bf16, void *dx_bf16) {
    const char *fn = "pcnn_dwconv_dgrad";
    PCNN_REQUIRE(ctx && plan && dy_bf16 && dx_bf16, PCNN_ERR_ARG, "%s: NULL argument", fn);
    DwConvPlan *pl;
    int rc = plan_as(fn, plan, &pl);
    if (rc) return rc;
    PCNN_REQUIRE(aligned16(dy_bf16) && aligned16(dx_bf16), PCNN_ERR_ARG, "%s: dy and dx must be 16-byte aligned", fn);
    const DwArgs &a = pl->a;
    const size_t xb = (size_t)a.N * a.H * a.W * a.C * 2, yb = (size_t)a.M * a.C * 2;
    PCNN_REQUIRE(!overlap(dx_bf16, xb, dy_bf16, yb), PCNN_ERR_ARG, "%s: overlapping buffers: dy and dx must not share memory", fn);
    pcnn_device_guard g(ctx->device);
    const dim3 grid((unsigned)((a.dstrips + a.lanes - 1) / a.lanes), (unsigned)a.slices);
    const auto *dy = static_cast<const __nv_bfloat16 *>(dy_bf16);
    auto *dx = static_cast<__nv_bfloat16 *>(dx_bf16);
    const bool dil = a.dil_h > 1 || a.dil_w > 1;
    if (a.C % 8 == 0)
        (dil ? k_dwconv_dgrad<8, true> : k_dwconv_dgrad<8, false>)<<<grid, DW_THREADS, 0, ctx->stream>>>(dy, pl->wop(), dx, a);
    else
        (dil ? k_dwconv_dgrad<1, true> : k_dwconv_dgrad<1, false>)<<<grid, DW_THREADS, 0, ctx->stream>>>(dy, pl->wop(), dx, a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
