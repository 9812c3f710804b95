// parallel-cnn_b200/csrc/regress_loss.cu -- per-element regression losses for device-trained networks (pcnn_regression_loss_bf16):
// mean squared error and mean absolute error of a dense bf16 prediction [pixels][C] against the first C channels of a bf16 target
// [pixels][target_stride], the gradient dpred at a caller-chosen scale and the unscaled loss of every pixel.  The fp32 operations
// and their order are include/pcnn.h's.  The binary cross-entropy with logits (pcnn_bce_logits_bf16) runs its own kernel on the
// same layout and partition.
//
// One CTA per tile of RL_TILE pixels, walking the channels in chunks of at most RL_CHUNK: each thread takes VEC consecutive
// channels of one pixel (VEC = 8, 16-byte accesses, when C and target_stride are multiples of 8), writes their dpred and leaves
// their loss terms in shared memory; then one thread per pixel adds its terms in ascending channel order.  No cross-CTA
// reduction and no atomics, so every bit is independent of the grid and of reruns.
#include "pcnn_internal.h"

#include <cuda_bf16.h>

#include <cmath>

namespace {

constexpr int RL_THREADS = 256;
constexpr int RL_TILE = 64;                  // pixels per CTA
constexpr int RL_CHUNK = 120;                // channels per pass over shared memory (a multiple of 8)

struct RlArgs {
    const __nv_bfloat16 *pred, *target;
    __nv_bfloat16 *dpred;
    float *loss;
    long long pixels;
    int C, ts, mode;
    float scale;
};

template <int VEC>
struct alignas(2 * VEC) Bf16Vec {
    __nv_bfloat16 v[VEC];
};

// the sign that multiplies the L1 gradient's scale: +0 at d = +-0 and at NaN, as torch's sign
__device__ __forceinline__ float l1_sign(float d) { return d > 0.0f ? 1.0f : d < 0.0f ? -1.0f : 0.0f; }

template <int VEC>
__global__ void __launch_bounds__(RL_THREADS) k_regression_loss(const RlArgs a) {
    __shared__ float terms[RL_TILE][RL_CHUNK + 1];
    const long long p0 = (long long)blockIdx.x * RL_TILE;
    const int np = (int)min((long long)RL_TILE, a.pixels - p0);
    const float k2 = __fmul_rn(2.0f, a.scale);
    float s = 0.0f;                                          // thread p < np: the running loss of pixel p0 + p
    for (int c0 = 0; c0 < a.C; c0 += RL_CHUNK) {
        const int cc = min(RL_CHUNK, a.C - c0), G = cc / VEC;
        for (int v = threadIdx.x; v < np * G; v += RL_THREADS) {
            const int p = v / G, cl = (v - p * G) * VEC;
            const long long px = p0 + p;
            const Bf16Vec<VEC> pv = *reinterpret_cast<const Bf16Vec<VEC> *>(a.pred + px * a.C + c0 + cl);
            const Bf16Vec<VEC> tv = *reinterpret_cast<const Bf16Vec<VEC> *>(a.target + px * a.ts + c0 + cl);
            Bf16Vec<VEC> g;
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                const float d = __fsub_rn(__bfloat162float(pv.v[k]), __bfloat162float(tv.v[k]));
                float term, grad;
                if (a.mode == PCNN_LOSS_MSE) {
                    term = __fmul_rn(d, d);
                    grad = __fmul_rn(k2, d);
                } else {
                    term = fabsf(d);
                    grad = __fmul_rn(l1_sign(d), a.scale);
                }
                g.v[k] = __float2bfloat16_rn(grad);
                terms[p][cl + k] = term;
            }
            *reinterpret_cast<Bf16Vec<VEC> *>(a.dpred + px * a.C + c0 + cl) = g;
        }
        if (a.loss) {
            __syncthreads();
            if (threadIdx.x < np)
                for (int c = 0; c < cc; ++c) s = __fadd_rn(s, terms[threadIdx.x][c]);
            __syncthreads();
        }
    }
    if (a.loss && threadIdx.x < np) a.loss[p0 + threadIdx.x] = s;
}

// binary cross-entropy with logits on the same tile layout: each element's loss term max(x, 0) - x t + log1p(E(-|x|)) and
// gradient scale (sigma(x) - t), sigma = 1 / (1 + e) (x >= 0) or e / (1 + e) (x < 0) with e = E(-|x|), so neither overflows
template <int VEC>
__global__ void __launch_bounds__(RL_THREADS) k_bce_logits(const RlArgs a) {
    __shared__ float terms[RL_TILE][RL_CHUNK + 1];
    const long long p0 = (long long)blockIdx.x * RL_TILE;
    const int np = (int)min((long long)RL_TILE, a.pixels - p0);
    float s = 0.0f;                                          // thread p < np: the running loss of pixel p0 + p
    for (int c0 = 0; c0 < a.C; c0 += RL_CHUNK) {
        const int cc = min(RL_CHUNK, a.C - c0), G = cc / VEC;
        for (int v = threadIdx.x; v < np * G; v += RL_THREADS) {
            const int p = v / G, cl = (v - p * G) * VEC;
            const long long px = p0 + p;
            const Bf16Vec<VEC> xv = *reinterpret_cast<const Bf16Vec<VEC> *>(a.pred + px * a.C + c0 + cl);
            const Bf16Vec<VEC> tv = *reinterpret_cast<const Bf16Vec<VEC> *>(a.target + px * a.ts + c0 + cl);
            Bf16Vec<VEC> g;
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                const float x = __bfloat162float(xv.v[k]), t = __bfloat162float(tv.v[k]);
                const float e = exp_f32(-fabsf(x));
                const float term = __fadd_rn(__fsub_rn(x > 0.0f ? x : 0.0f, __fmul_rn(x, t)), log1p_f32(e));
                const float sig = __fdiv_rn(x >= 0.0f ? 1.0f : e, __fadd_rn(1.0f, e));
                g.v[k] = __float2bfloat16_rn(__fmul_rn(a.scale, __fsub_rn(sig, t)));
                terms[p][cl + k] = term;
            }
            *reinterpret_cast<Bf16Vec<VEC> *>(a.dpred + px * a.C + c0 + cl) = g;
        }
        if (a.loss) {
            __syncthreads();
            if (threadIdx.x < np)
                for (int c = 0; c < cc; ++c) s = __fadd_rn(s, terms[threadIdx.x][c]);
            __syncthreads();
        }
    }
    if (a.loss && threadIdx.x < np) a.loss[p0 + threadIdx.x] = s;
}

bool rl_disjoint(const void *a, size_t abytes, const void *b, size_t bbytes) {
    const uintptr_t pa = (uintptr_t)a, pb = (uintptr_t)b;
    return pa + abytes <= pb || pb + bbytes <= pa;
}

}  // namespace

extern "C" int pcnn_regression_loss_bf16(pcnn_ctx *ctx, const void *pred_bf16_dev, const void *target_bf16_dev, int target_stride,
                                         int pixels, int C, int mode, float scale, void *dpred_bf16_dev, float *loss_f32_dev) {
    const char *fn = "pcnn_regression_loss_bf16";
    PCNN_REQUIRE(ctx && pred_bf16_dev && target_bf16_dev && dpred_bf16_dev, PCNN_ERR_ARG, "%s: NULL argument", fn);
    PCNN_REQUIRE(pixels >= 1, PCNN_ERR_ARG, "%s: pixels = %d: at least 1 is required", fn, pixels);
    PCNN_REQUIRE(C >= 1 && C <= target_stride, PCNN_ERR_ARG, "%s: C = %d, target_stride = %d: 1 <= C <= target_stride is required", fn,
                 C, target_stride);
    PCNN_REQUIRE(mode == PCNN_LOSS_MSE || mode == PCNN_LOSS_L1, PCNN_ERR_ARG, "%s: mode %d is not 0 (MSE) or 1 (L1)", fn, mode);
    PCNN_REQUIRE(std::isfinite(scale), PCNN_ERR_ARG, "%s: scale = %g: a finite scale is required", fn, (double)scale);
    PCNN_REQUIRE((((uintptr_t)pred_bf16_dev | (uintptr_t)target_bf16_dev | (uintptr_t)dpred_bf16_dev | (uintptr_t)loss_f32_dev) & 15) == 0,
                 PCNN_ERR_ARG, "%s: pred, target, dpred and loss must be 16-byte aligned", fn);
    const size_t pbytes = (size_t)pixels * C * 2, tbytes = ((size_t)(pixels - 1) * target_stride + C) * 2, lbytes = (size_t)pixels * 4;
    PCNN_REQUIRE(dpred_bf16_dev == pred_bf16_dev || rl_disjoint(dpred_bf16_dev, pbytes, pred_bf16_dev, pbytes), PCNN_ERR_ARG,
                 "%s: dpred overlaps pred without being pred: only dpred == pred (in place) is allowed", fn);
    PCNN_REQUIRE(rl_disjoint(dpred_bf16_dev, pbytes, target_bf16_dev, tbytes), PCNN_ERR_ARG, "%s: dpred overlaps target", fn);
    PCNN_REQUIRE(!loss_f32_dev || (rl_disjoint(loss_f32_dev, lbytes, pred_bf16_dev, pbytes) &&
                                   rl_disjoint(loss_f32_dev, lbytes, target_bf16_dev, tbytes) &&
                                   rl_disjoint(loss_f32_dev, lbytes, dpred_bf16_dev, pbytes)),
                 PCNN_ERR_ARG, "%s: loss overlaps pred, target or dpred", fn);
    pcnn_device_guard g(ctx->device);
    RlArgs a;
    a.pred = static_cast<const __nv_bfloat16 *>(pred_bf16_dev);
    a.target = static_cast<const __nv_bfloat16 *>(target_bf16_dev);
    a.dpred = static_cast<__nv_bfloat16 *>(dpred_bf16_dev);
    a.loss = loss_f32_dev;
    a.pixels = pixels;
    a.C = C;
    a.ts = target_stride;
    a.mode = mode;
    a.scale = scale;
    const unsigned grid = (unsigned)((pixels + (long long)RL_TILE - 1) / RL_TILE);
    if (C % 8 == 0 && target_stride % 8 == 0) k_regression_loss<8><<<grid, RL_THREADS, 0, ctx->stream>>>(a);
    else k_regression_loss<1><<<grid, RL_THREADS, 0, ctx->stream>>>(a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_bce_logits_bf16(pcnn_ctx *ctx, const void *logits_bf16_dev, const void *target_bf16_dev, int target_stride,
                                    int pixels, int C, float scale, void *dlogits_bf16_dev, float *loss_f32_dev) {
    const char *fn = "pcnn_bce_logits_bf16";
    PCNN_REQUIRE(ctx && logits_bf16_dev && target_bf16_dev && dlogits_bf16_dev, PCNN_ERR_ARG, "%s: NULL argument", fn);
    PCNN_REQUIRE(pixels >= 1, PCNN_ERR_ARG, "%s: pixels = %d: at least 1 is required", fn, pixels);
    PCNN_REQUIRE(C >= 1 && C <= target_stride, PCNN_ERR_ARG, "%s: C = %d, target_stride = %d: 1 <= C <= target_stride is required", fn,
                 C, target_stride);
    PCNN_REQUIRE(std::isfinite(scale), PCNN_ERR_ARG, "%s: scale = %g: a finite scale is required", fn, (double)scale);
    PCNN_REQUIRE((((uintptr_t)logits_bf16_dev | (uintptr_t)target_bf16_dev | (uintptr_t)dlogits_bf16_dev | (uintptr_t)loss_f32_dev) & 15) ==
                     0,
                 PCNN_ERR_ARG, "%s: logits, target, dlogits and loss must be 16-byte aligned", fn);
    const size_t pbytes = (size_t)pixels * C * 2, tbytes = ((size_t)(pixels - 1) * target_stride + C) * 2, lbytes = (size_t)pixels * 4;
    PCNN_REQUIRE(dlogits_bf16_dev == logits_bf16_dev || rl_disjoint(dlogits_bf16_dev, pbytes, logits_bf16_dev, pbytes), PCNN_ERR_ARG,
                 "%s: dlogits overlaps logits without being logits: only dlogits == logits (in place) is allowed", fn);
    PCNN_REQUIRE(rl_disjoint(dlogits_bf16_dev, pbytes, target_bf16_dev, tbytes), PCNN_ERR_ARG, "%s: dlogits overlaps target", fn);
    PCNN_REQUIRE(!loss_f32_dev || (rl_disjoint(loss_f32_dev, lbytes, logits_bf16_dev, pbytes) &&
                                   rl_disjoint(loss_f32_dev, lbytes, target_bf16_dev, tbytes) &&
                                   rl_disjoint(loss_f32_dev, lbytes, dlogits_bf16_dev, pbytes)),
                 PCNN_ERR_ARG, "%s: loss overlaps logits, target or dlogits", fn);
    pcnn_device_guard g(ctx->device);
    RlArgs a;
    a.pred = static_cast<const __nv_bfloat16 *>(logits_bf16_dev);
    a.target = static_cast<const __nv_bfloat16 *>(target_bf16_dev);
    a.dpred = static_cast<__nv_bfloat16 *>(dlogits_bf16_dev);
    a.loss = loss_f32_dev;
    a.pixels = pixels;
    a.C = C;
    a.ts = target_stride;
    a.mode = 0;
    a.scale = scale;
    const unsigned grid = (unsigned)((pixels + (long long)RL_TILE - 1) / RL_TILE);
    if (C % 8 == 0 && target_stride % 8 == 0) k_bce_logits<8><<<grid, RL_THREADS, 0, ctx->stream>>>(a);
    else k_bce_logits<1><<<grid, RL_THREADS, 0, ctx->stream>>>(a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
