// parallel-cnn_b200/csrc/upsample_nhwc.cu -- bilinear resizing between device-trained layers (pcnn_upsample_bilinear_nhwc_bf16_fwd /
// _bwd and the host-only pcnn_upsample_bilinear_info), as torch.nn.functional.interpolate(size=(H_out, W_out), mode="bilinear",
// align_corners=False) on dense NHWC bf16 maps.  The source index and the weights of every output row and column are formed in fp32
// by the rule include/pcnn.h states, the same in both passes.
//
// Forward: one thread per (output pixel, group of VEC channels) reads the four source pixels and writes one bf16 result.
// Backward: a gather, no atomics.  One thread per (input pixel, group of VEC channels) finds the output rows whose taps reach its
// row (the first tap's index is monotone in the output row, so a binary search finds the first; the walk stops past the last) and
// the same for columns, and sums their weighted dy in a fixed order in fp32 before one bf16 rounding: reruns give the same bits.
#include "pcnn_internal.h"

#include <cuda_bf16.h>

#include <climits>

namespace {

constexpr int UP_THREADS = 256;
constexpr int UP_MAX_SIDE = 16384;        // dst + 0.5 and every index stay exact in fp32
constexpr long long UP_MAX_GRID = 1 << 20;

// One axis: in -> out.  scale = RN32(in / out).  Output index d reads source indices i0, i1 with weights l0, l1:
//   in == out: i0 = i1 = d, l0 = 1, l1 = 0 (per axis, as torch's CPU kernel; its CUDA kernel copies only when both axes are);
//   else real = RN(RN(scale * RN(d + 0.5)) - 0.5), real = real < 0 ? 0 : real; i0 = min(floor(real), in - 1);
//        l1 = min(max(RN(real - i0), 0), 1); l0 = RN(1 - l1); i1 = i0 + (i0 < in - 1).
struct Axis {
    int in, out;
    float scale;
};

struct Tap {
    int i0, i1;
    float l0, l1;
};

__device__ __forceinline__ Tap axis_tap(const Axis &a, int d) {
    Tap t;
    if (a.in == a.out) {
        t.i0 = t.i1 = d;
        t.l0 = 1.0f;
        t.l1 = 0.0f;
        return t;
    }
    float real = __fsub_rn(__fmul_rn(a.scale, __fadd_rn((float)d, 0.5f)), 0.5f);
    real = real < 0.0f ? 0.0f : real;
    int i0 = (int)floorf(real);
    i0 = i0 < a.in - 1 ? i0 : a.in - 1;
    float l1 = __fsub_rn(real, (float)i0);
    l1 = fminf(fmaxf(l1, 0.0f), 1.0f);
    t.i0 = i0;
    t.i1 = i0 + (i0 < a.in - 1 ? 1 : 0);
    t.l1 = l1;
    t.l0 = __fsub_rn(1.0f, l1);
    return t;
}

// the first output index whose first tap is >= i (out when none)
__device__ __forceinline__ int first_reaching(const Axis &a, int i) {
    int lo = 0, hi = a.out;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (axis_tap(a, mid).i0 >= i) hi = mid; else lo = mid + 1;
    }
    return lo;
}

// the weight with which output index d's taps reach source index i, or false when neither tap is i: l0 and l1 added in fp32 when
// both taps are i (the clamped last index)
__device__ __forceinline__ bool tap_weight(const Tap &t, int i, float &w) {
    if (t.i0 == i && t.i1 == i) { w = __fadd_rn(t.l0, t.l1); return true; }
    if (t.i0 == i) { w = t.l0; return true; }
    if (t.i1 == i) { w = t.l1; return true; }
    return false;
}

struct UpArgs {
    const __nv_bfloat16 *src;   // forward: x [N][H][W][C]; backward: dy [N][H_out][W_out][C]
    __nv_bfloat16 *dst;         // forward: y; backward: dx
    int N, C, G;                // G = C / VEC groups of channels
    Axis h, w;
    long long total;            // threads' items: N * (rows) * (cols) * G of the destination
};

template <int VEC>
struct alignas(2 * VEC) Bf16Vec {
    __nv_bfloat16 v[VEC];
};

// y = bf16_rn(RN(RN(lh0 * top) + RN(lh1 * bot))), top = RN(RN(lw0 * x[i0][j0]) + RN(lw1 * x[i0][j1])), bot the same on row i1
template <int VEC>
__global__ void __launch_bounds__(UP_THREADS) k_upsample_fwd(const UpArgs a) {
    for (long long t = blockIdx.x * (long long)UP_THREADS + threadIdx.x; t < a.total; t += (long long)gridDim.x * UP_THREADS) {
        const int g = (int)(t % a.G);
        long long r = t / a.G;
        const int ow = (int)(r % a.w.out);
        r /= a.w.out;
        const int oh = (int)(r % a.h.out);
        const long long n = r / a.h.out;
        const Tap th = axis_tap(a.h, oh), tw = axis_tap(a.w, ow);
        const __nv_bfloat16 *img = a.src + n * a.h.in * (long long)a.w.in * a.C + (long long)g * VEC;
        const Bf16Vec<VEC> x00 = *reinterpret_cast<const Bf16Vec<VEC> *>(img + ((long long)th.i0 * a.w.in + tw.i0) * a.C);
        const Bf16Vec<VEC> x01 = *reinterpret_cast<const Bf16Vec<VEC> *>(img + ((long long)th.i0 * a.w.in + tw.i1) * a.C);
        const Bf16Vec<VEC> x10 = *reinterpret_cast<const Bf16Vec<VEC> *>(img + ((long long)th.i1 * a.w.in + tw.i0) * a.C);
        const Bf16Vec<VEC> x11 = *reinterpret_cast<const Bf16Vec<VEC> *>(img + ((long long)th.i1 * a.w.in + tw.i1) * a.C);
        Bf16Vec<VEC> y;
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            const float top = __fadd_rn(__fmul_rn(tw.l0, __bfloat162float(x00.v[k])), __fmul_rn(tw.l1, __bfloat162float(x01.v[k])));
            const float bot = __fadd_rn(__fmul_rn(tw.l0, __bfloat162float(x10.v[k])), __fmul_rn(tw.l1, __bfloat162float(x11.v[k])));
            y.v[k] = __float2bfloat16_rn(__fadd_rn(__fmul_rn(th.l0, top), __fmul_rn(th.l1, bot)));
        }
        *reinterpret_cast<Bf16Vec<VEC> *>(a.dst + t * VEC) = y;
    }
}

// dx[n][i][j][c] = bf16_rn(s), s the fp32 sum from +0 over the output rows oh ascending, then the output columns ow ascending,
// whose taps reach (i, j), of RN(RN(wh * ww) * dy[n][oh][ow][c]) with wh, ww tap_weight's
template <int VEC>
__global__ void __launch_bounds__(UP_THREADS) k_upsample_bwd(const UpArgs a) {
    for (long long t = blockIdx.x * (long long)UP_THREADS + threadIdx.x; t < a.total; t += (long long)gridDim.x * UP_THREADS) {
        const int g = (int)(t % a.G);
        long long r = t / a.G;
        const int j = (int)(r % a.w.in);
        r /= a.w.in;
        const int i = (int)(r % a.h.in);
        const long long n = r / a.h.in;
        const __nv_bfloat16 *img = a.src + n * a.h.out * (long long)a.w.out * a.C + (long long)g * VEC;
        float s[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) s[k] = 0.0f;
        const int oh0 = first_reaching(a.h, i - 1), ow0 = first_reaching(a.w, j - 1);
        for (int oh = oh0; oh < a.h.out; ++oh) {
            const Tap th = axis_tap(a.h, oh);
            if (th.i0 > i) break;
            float wh;
            if (!tap_weight(th, i, wh)) continue;
            for (int ow = ow0; ow < a.w.out; ++ow) {
                const Tap tw = axis_tap(a.w, ow);
                if (tw.i0 > j) break;
                float ww;
                if (!tap_weight(tw, j, ww)) continue;
                const float wt = __fmul_rn(wh, ww);
                const Bf16Vec<VEC> d = *reinterpret_cast<const Bf16Vec<VEC> *>(img + ((long long)oh * a.w.out + ow) * a.C);
#pragma unroll
                for (int k = 0; k < VEC; ++k) s[k] = __fadd_rn(s[k], __fmul_rn(wt, __bfloat162float(d.v[k])));
            }
        }
        Bf16Vec<VEC> o;
#pragma unroll
        for (int k = 0; k < VEC; ++k) o.v[k] = __float2bfloat16_rn(s[k]);
        *reinterpret_cast<Bf16Vec<VEC> *>(a.dst + t * VEC) = o;
    }
}

struct UpShape {
    UpArgs fwd, bwd;
    int vec;
    long long grid_fwd, grid_bwd;
};

int up_shape(const char *fn, int N, int H, int W, int C, int H_out, int W_out, UpShape *s) {
    PCNN_REQUIRE(N >= 1 && C >= 1, PCNN_ERR_ARG, "%s: N = %d, C = %d: each must be >= 1", fn, N, C);
    PCNN_REQUIRE(H >= 1 && W >= 1 && H_out >= 1 && W_out >= 1, PCNN_ERR_ARG,
                 "%s: H = %d, W = %d, H_out = %d, W_out = %d: each must be >= 1", fn, H, W, H_out, W_out);
    PCNN_REQUIRE(H <= UP_MAX_SIDE && W <= UP_MAX_SIDE && H_out <= UP_MAX_SIDE && W_out <= UP_MAX_SIDE, PCNN_ERR_ARG,
                 "%s: H = %d, W = %d, H_out = %d, W_out = %d: each side must be <= %d", fn, H, W, H_out, W_out, UP_MAX_SIDE);
    const double big = (double)N * C * ((double)H * W > (double)H_out * W_out ? (double)H * W : (double)H_out * W_out);
    PCNN_REQUIRE(big * 2.0 < 4611686018427387904.0, PCNN_ERR_ARG, "%s: N H W C = %.0f elements: each map must be below 2^62 bytes",
                 fn, big);
    s->vec = C % 8 == 0 ? 8 : 1;
    UpArgs a;
    memset(&a, 0, sizeof(a));
    a.N = N;
    a.C = C;
    a.G = C / s->vec;
    a.h = Axis{H, H_out, (float)H / (float)H_out};
    a.w = Axis{W, W_out, (float)W / (float)W_out};
    s->fwd = a;
    s->fwd.total = (long long)N * H_out * W_out * a.G;
    s->bwd = a;
    s->bwd.total = (long long)N * H * W * a.G;
    auto grid = [](long long items) {
        const long long g = (items + UP_THREADS - 1) / UP_THREADS;
        return g < UP_MAX_GRID ? g : UP_MAX_GRID;
    };
    s->grid_fwd = grid(s->fwd.total);
    s->grid_bwd = grid(s->bwd.total);
    return PCNN_OK;
}

bool up_disjoint(const void *a, size_t abytes, const void *b, size_t bbytes) {
    const uintptr_t pa = (uintptr_t)a, pb = (uintptr_t)b;
    return pa + abytes <= pb || pb + bbytes <= pa;
}

int up_run(const char *fn, pcnn_ctx *ctx, const void *src, void *dst, int N, int H, int W, int C, int H_out, int W_out, bool bwd) {
    PCNN_REQUIRE(ctx && src && dst, PCNN_ERR_ARG, "%s: NULL argument", fn);
    UpShape s;
    int rc = up_shape(fn, N, H, W, C, H_out, W_out, &s);
    if (rc) return rc;
    PCNN_REQUIRE(s.vec == 1 || (((uintptr_t)src | (uintptr_t)dst) & 15) == 0, PCNN_ERR_ARG,
                 "%s: with C %% 8 == 0 both maps must be 16-byte aligned", fn);
    const size_t small = (size_t)N * H * W * C * 2, large = (size_t)N * H_out * W_out * C * 2;
    PCNN_REQUIRE(up_disjoint(src, bwd ? large : small, dst, bwd ? small : large), PCNN_ERR_ARG, "%s: the two maps overlap", fn);
    pcnn_device_guard g(ctx->device);
    const UpArgs &a = bwd ? s.bwd : s.fwd;
    UpArgs aa = a;
    aa.src = static_cast<const __nv_bfloat16 *>(src);
    aa.dst = static_cast<__nv_bfloat16 *>(dst);
    const unsigned grid = (unsigned)(bwd ? s.grid_bwd : s.grid_fwd);
    if (bwd) {
        if (s.vec == 8) k_upsample_bwd<8><<<grid, UP_THREADS, 0, ctx->stream>>>(aa);
        else k_upsample_bwd<1><<<grid, UP_THREADS, 0, ctx->stream>>>(aa);
    } else {
        if (s.vec == 8) k_upsample_fwd<8><<<grid, UP_THREADS, 0, ctx->stream>>>(aa);
        else k_upsample_fwd<1><<<grid, UP_THREADS, 0, ctx->stream>>>(aa);
    }
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

}  // namespace

extern "C" int pcnn_upsample_bilinear_info(int N, int H, int W, int C, int H_out, int W_out, long long *out4) {
    const char *fn = "pcnn_upsample_bilinear_info";
    PCNN_REQUIRE(out4, PCNN_ERR_ARG, "%s: NULL out4", fn);
    UpShape s;
    const int rc = up_shape(fn, N, H, W, C, H_out, W_out, &s);
    if (rc) return rc;
    out4[0] = s.vec;
    out4[1] = s.grid_fwd;
    out4[2] = s.grid_bwd;
    out4[3] = UP_THREADS;
    return PCNN_OK;
}

extern "C" int pcnn_upsample_bilinear_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, void *y_bf16_dev, int N, int H, int W, int C,
                                                    int H_out, int W_out) {
    return up_run("pcnn_upsample_bilinear_nhwc_bf16_fwd", ctx, x_bf16_dev, y_bf16_dev, N, H, W, C, H_out, W_out, false);
}

extern "C" int pcnn_upsample_bilinear_nhwc_bf16_bwd(pcnn_ctx *ctx, const void *dy_bf16_dev, void *dx_bf16_dev, int N, int H, int W, int C,
                                                    int H_out, int W_out) {
    return up_run("pcnn_upsample_bilinear_nhwc_bf16_bwd", ctx, dy_bf16_dev, dx_bf16_dev, N, H, W, C, H_out, W_out, true);
}
