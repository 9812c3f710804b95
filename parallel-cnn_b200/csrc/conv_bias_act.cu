// parallel-cnn_b200/csrc/conv_bias_act.cu -- the gradient at the pre-activation and the bias gradient of a convolution or linear
// layer (pcnn_conv_bias_act_bwd), in one pass over dy:
//     dpre = bf16_rn(dy * (y * (1 - y)))      (act 1: y is the sigmoid output the forward stored; fp32, no contraction)
//     dpre = float(y) <= 0 ? +0 : dy          (act 3: y is the ReLU output; dy's bits pass through, a NaN y passes dy)
//     db[k] = sum over pixels of float(dpre[pixel][k])      (of dy at act 0)
// so db sums exactly the bf16 values the weight and input gradients consume.
//
// The pass is HBM-bound (read y and dy, write dpre: the same bytes at act 1 and 3).  With K % 8 == 0 a thread moves 16-byte
// vectors of 8 channels of one pixel, otherwise single elements.  A CTA owns the fixed pixel range
// [b * BA_ITERS * lanes, (b + 1) * BA_ITERS * lanes): thread t keeps channel group g = t % G of pixel lane t / G (G = K / VEC groups, lanes = 256 / G), so its VEC accumulators
// stay on the same channels over its BA_ITERS pixels, which are loaded before any is stored (in place, dpre == dy, each element
// is read and written by one thread).  The lanes' sums go through shared memory into the CTA's slot [b][K] in lane order, and
// pcnn_conv_wgrad_reduce_slots adds the slots in a fixed order.  Nothing depends on the SM count: the bits of db are the same
// on every run and every H100.
#include "pcnn_internal.h"

#include <cuda_bf16.h>

namespace {

constexpr int BA_THREADS = 256;
constexpr int BA_ITERS = 8;          // pixels per thread

template <int VEC>
struct alignas(2 * VEC) BfVec {
    __nv_bfloat16 h[VEC];
};

template <int VEC, int ACT>
__global__ void __launch_bounds__(BA_THREADS) k_conv_bias_act_bwd(const __nv_bfloat16 *y, const __nv_bfloat16 *dy, __nv_bfloat16 *dpre,
                                                                  float *slots, long pixels, int K) {
    __shared__ float part[BA_THREADS * VEC];         // [lanes][K]: lanes * K <= 256 * VEC
    const int G = K / VEC, lanes = BA_THREADS / G;
    const int lane = threadIdx.x / G, g = threadIdx.x % G;
    float acc[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = 0.0f;
    if (lane < lanes) {
        const long px0 = (long)blockIdx.x * BA_ITERS * lanes + lane;
        BfVec<VEC> gv[BA_ITERS], yv[BA_ITERS];
#pragma unroll
        for (int j = 0; j < BA_ITERS; ++j) {
            const long px = px0 + (long)j * lanes;
            if (px < pixels) {
                const long off = px * K + g * VEC;
                gv[j] = *reinterpret_cast<const BfVec<VEC> *>(dy + off);
                if (ACT) yv[j] = *reinterpret_cast<const BfVec<VEC> *>(y + off);
            }
        }
#pragma unroll
        for (int j = 0; j < BA_ITERS; ++j) {
            const long px = px0 + (long)j * lanes;
            if (px < pixels) {
                BfVec<VEC> d = gv[j];
                if (ACT) {
#pragma unroll
                    for (int i = 0; i < VEC; ++i) {
                        const float yf = __bfloat162float(yv[j].h[i]);
                        if (ACT == PCNN_ACT_SIGMOID) {
                            const float gf = __bfloat162float(gv[j].h[i]);
                            d.h[i] = __float2bfloat16_rn(__fmul_rn(gf, __fmul_rn(yf, __fsub_rn(1.0f, yf))));
                        }
                        else if (yf <= 0.0f)                     // ReLU: d keeps dy's bits where y > 0 or NaN
                            d.h[i] = __ushort_as_bfloat16((unsigned short)0);
                    }
                    *reinterpret_cast<BfVec<VEC> *>(dpre + px * K + g * VEC) = d;
                }
#pragma unroll
                for (int i = 0; i < VEC; ++i) acc[i] = __fadd_rn(acc[i], __bfloat162float(d.h[i]));
            }
        }
    }
    if (!slots) return;                              // no bias: dpre only
    if (lane < lanes)
#pragma unroll
        for (int i = 0; i < VEC; ++i) part[lane * K + g * VEC + i] = acc[i];
    __syncthreads();
    if (threadIdx.x < K) {
        float s = 0.0f;
        for (int l = 0; l < lanes; ++l) s = __fadd_rn(s, part[l * K + threadIdx.x]);
        slots[(long)blockIdx.x * K + threadIdx.x] = s;
    }
}

typedef void (*bias_act_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, __nv_bfloat16 *, float *, long, int);

bool overlap(const void *a, size_t na, const void *b, size_t nb) {
    if (!a || !b) return false;
    const uintptr_t pa = (uintptr_t)a, pb = (uintptr_t)b;
    return pa < pb + nb && pb < pa + na;
}

}  // namespace

extern "C" int pcnn_conv_bias_act_bwd(pcnn_ctx *ctx, const void *y_bf16, const void *dy_bf16, void *dpre_bf16, float *db_f32, long pixels,
                                      int K, int act) {
    const char *fn = "pcnn_conv_bias_act_bwd";
    PCNN_REQUIRE(ctx && dy_bf16, PCNN_ERR_ARG, "%s: NULL context or dy", fn);
    PCNN_REQUIRE_ACT(fn, act);
    PCNN_REQUIRE(K >= 1 && K <= 256, PCNN_ERR_ARG, "%s: K = %d filters: 1 <= K <= 256 is required", fn, K);
    PCNN_REQUIRE(pixels >= 1, PCNN_ERR_ARG, "%s: pixels = %ld: at least one pixel (N * P * Q) is required", fn, pixels);
    if (act != PCNN_ACT_NONE)
        PCNN_REQUIRE(y_bf16 && dpre_bf16, PCNN_ERR_ARG, "%s: act %d (%s) needs y, the forward's output, and dpre (NULL given)", fn,
                     act, act == PCNN_ACT_SIGMOID ? "sigmoid" : "ReLU");
    else
        PCNN_REQUIRE(!dpre_bf16 && db_f32, PCNN_ERR_ARG,
                     "%s: act 0 writes no dpre (it must be NULL) and computes db only (it must not be NULL)", fn);
    const void *y = act != PCNN_ACT_NONE ? y_bf16 : nullptr;
    const void *ptrs[4] = {y, dy_bf16, dpre_bf16, db_f32};
    for (const void *q : ptrs)
        PCNN_REQUIRE(((uintptr_t)q & 15) == 0, PCNN_ERR_ARG, "%s: y, dy, dpre and db must be 16-byte aligned", fn);
    const size_t bytes = (size_t)pixels * K * 2, db_bytes = (size_t)K * sizeof(float);
    PCNN_REQUIRE((dpre_bf16 == dy_bf16 || !overlap(dpre_bf16, bytes, dy_bf16, bytes)) && !overlap(dpre_bf16, bytes, y, bytes) &&
                     !overlap(db_f32, db_bytes, y, bytes) && !overlap(db_f32, db_bytes, dy_bf16, bytes) &&
                     !overlap(db_f32, db_bytes, dpre_bf16, bytes),
                 PCNN_ERR_ARG, "%s: overlapping buffers: only dpre == dy (in place) may share memory", fn);
    pcnn_device_guard g(ctx->device);
    const bool vec = K % 8 == 0;
    const int lanes = BA_THREADS / (vec ? K / 8 : K);
    const long per_cta = (long)BA_ITERS * lanes;
    const long ctas = (pixels + per_cta - 1) / per_cta;
    PCNN_REQUIRE(ctas < (1L << 31), PCNN_ERR_ARG, "%s: %ld pixels exceed the grid", fn, pixels);
    float *slots = nullptr;
    if (db_f32) {
        int rc = pcnn_scratch(ctx, (size_t)ctas * K * sizeof(float), (void **)&slots);
        if (rc) return rc;
    }
    static const bias_act_fn table[2][3] = {
        {k_conv_bias_act_bwd<1, PCNN_ACT_NONE>, k_conv_bias_act_bwd<1, PCNN_ACT_SIGMOID>, k_conv_bias_act_bwd<1, PCNN_ACT_RELU>},
        {k_conv_bias_act_bwd<8, PCNN_ACT_NONE>, k_conv_bias_act_bwd<8, PCNN_ACT_SIGMOID>, k_conv_bias_act_bwd<8, PCNN_ACT_RELU>}};
    table[vec ? 1 : 0][pcnn_act_col(act)]<<<(unsigned)ctas, BA_THREADS, 0, ctx->stream>>>(
        static_cast<const __nv_bfloat16 *>(y), static_cast<const __nv_bfloat16 *>(dy_bf16), static_cast<__nv_bfloat16 *>(dpre_bf16),
        slots, pixels, K);
    PCNN_CHECK_LAUNCH(ctx);
    return db_f32 ? pcnn_conv_wgrad_reduce_slots(ctx, slots, db_f32, (int)ctas, K) : PCNN_OK;
}
