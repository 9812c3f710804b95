// parallel-cnn_b200/csrc/lenet5_kernels.cu -- the LeNet-5-style variant with a SECOND convolution layer (SURVEY.md 8f row 4;
// the reference has exactly one conv, Sequential/layer.h:105-140, net at Main.cpp:17-20):
//     28x28 -> c1 6@5x5 -> s2 shared 2x2/2 -> c3 16@5x5 over 6 channels -> s4 shared 2x2/2 -> f 256->10, sigmoid everywhere,
//     loss and update rules of the reference generalised by rule (oracle/lenet5_oracle.c states each rule and cites the
//     reference lines it extends).  PARITY UNPINNED by the reference: the checker is that self-written oracle.
// One fused kernel per step: a CTA runs forward + backward of its images with every activation and the 20.6 KB of
// parameters in shared memory (nothing but the 784-byte image crosses HBM per sample), per-CTA partial gradients,
// fixed-order slot reduction + update in a second kernel: deterministic, no atomics.
// The image pass is register-tiled and balanced phase by phase (see k_l5_step); the first version of this file (one thread per
// output, parameter-stationary gradient sums with up to 864-term serial chains) was bound by those serial chains.
#include "pcnn_internal.h"
#include "fused_body.cuh"

namespace {

constexpr int L5_T = 256;
constexpr int L5_NP = PCNN_L5_NPARAM;                 // 5152
constexpr int L5_NPK = L5_NP + 2;                     // + error-norm sum + pad
constexpr int L5_C1W = 0, L5_C1B = 150, L5_S2W = 156, L5_S2B = 160, L5_C3W = 161, L5_C3B = 2561, L5_S4W = 2577, L5_S4B = 2581,
              L5_FW = 2582, L5_FB = 5142;
constexpr int L5_ACC = (L5_NP + L5_T - 1) / L5_T;     // 21 packed entries per thread

struct L5Smem {
    alignas(16) float p[L5_NP + 4];
    alignas(16) float img[784];
    alignas(16) float c1o[3456];                      // [6][24][24]
    alignas(16) float s2o[864];                       // [6][12][12]
    alignas(16) float c3o[1024];                      // [16][8][8]
    alignas(16) float dpad[16 * 16 * 16];             // d_preact of c3, [16][8 + 8][8 + 8] with a zero border of 4 (the adjoint reads it unmasked)
    alignas(16) float dpre_s2[864];
    alignas(16) float red[216 * 27];                  // c1 weight-gradient partials of the 216 windows (+ bias sum), stride 27
    alignas(16) float gacc[L5_NP + 4];                // this CTA's batch sums of every entry but the f layer's (those live in registers)
    float dpre_s4[256];
    float fc_red[8][16];
    float part[8][8];                                 // per-warp partial sums of the subsample weight / bias gradients
    float fo[10];
};

struct L5Args {
    const void *images;
    const uint8_t *labels;
    const float *params;
    float *slots;          // [grid][L5_NPK]   (TRAIN)
    float *f_out;          // [B][10]          (EVAL)
    int B, pixel_u8;
};

using pcnn_fused::sigmoid_fast;
using pcnn_fused::warp_sum;
using pcnn_fused::warp_sum16_transposed;

// One image per CTA at a time, 256 threads, every phase register-tiled and balanced (no thread owns more than ~1,600 FMAs of a
// phase), activations in shared memory between phases:
//   c1 + s2      216 threads x (4 x 4 outputs of one map, the 8 x 8 patch in registers) -- the window tiling of fused_body.cuh
//   c3           256 threads x (map k, row x, 4 columns): 600 FMAs, input rows as 16-byte loads
//   s4, f        thread t owns s4 output t; f partial products reduced with the transposed warp sum
//   backward     f and s4 thread-local; d_preact of c3 into a zero-padded [16][16][16] array; c3 weight gradient: 480 items
//                (k, c, i) x 5 taps x 64 products; d_preact of s2 = adjoint of c3: 216 threads x 4 outputs x 400 FMAs over the
//                padded array (no masks); c1 weight gradient as in fused_body.cuh (per-window partials, then 36-way sums)
// Batch sums: the f layer's 2,570 entries in registers of their owner threads, everything else in S.gacc (each entry is
// touched by exactly one thread per image: no atomics, fixed order).
template <bool TRAIN> __global__ void __launch_bounds__(L5_T, 2) k_l5_step(const L5Args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    L5Smem &S = *reinterpret_cast<L5Smem *>(smem_raw);
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    for (int i = t; i < L5_NP; i += L5_T) S.p[i] = a.params[i];
    if (TRAIN) {
        for (int i = t; i < 16 * 16 * 16; i += L5_T) S.dpad[i] = 0.0f;
        for (int i = t; i < L5_NP + 4; i += L5_T) S.gacc[i] = 0.0f;
    }
    // roles
    const bool c1_worker = t < 216;
    const int m1 = c1_worker ? t / 36 : 0, wx = c1_worker ? (t % 36) / 6 : 0, wy = c1_worker ? t % 6 : 0;
    const int k3 = t >> 4, x3 = (t >> 1) & 7, h3 = t & 1;                    // c3: map, row, column half
    const int ms = t >> 4, xs = (t >> 2) & 3, ys = t & 3;                    // s4 output t
    const int c2 = c1_worker ? t / 36 : 0, u2 = c1_worker ? (t % 36) / 3 : 0, g2 = c1_worker ? t % 3 : 0;   // d_preact of s2
    float gfw[10], gfb = 0.0f, err_acc = 0.0f;
#pragma unroll
    for (int q = 0; q < 10; ++q) gfw[q] = 0.0f;

    for (int b = blockIdx.x; b < a.B; b += gridDim.x) {
        __syncthreads();                                   // parameters resident / previous image fully consumed
        // ---- image: (float)((double)u / 255.0) (mnist.h:145 + Main.cpp:64; one fp32 division rounds identically)
        if (a.pixel_u8) {
            const uint8_t *src = reinterpret_cast<const uint8_t *>(a.images) + (size_t)b * 784;
            for (int i = t; i < 196; i += L5_T) {
                const uchar4 q = reinterpret_cast<const uchar4 *>(src)[i];
                reinterpret_cast<float4 *>(S.img)[i] = make_float4(__fdiv_rn((float)q.x, 255.0f), __fdiv_rn((float)q.y, 255.0f),
                                                                   __fdiv_rn((float)q.z, 255.0f), __fdiv_rn((float)q.w, 255.0f));
            }
        } else {
            const float4 *src = reinterpret_cast<const float4 *>(reinterpret_cast<const float *>(a.images) + (size_t)b * 784);
            for (int i = t; i < 196; i += L5_T) reinterpret_cast<float4 *>(S.img)[i] = src[i];
        }
        const int label = TRAIN ? (int)a.labels[b] : 0;
        __syncthreads();

        // ---- c1 + sigmoid (layer.h:105-140) and s2 (rule of layer.h:143-181) for this thread's 4 x 4 window
        const float *ip = S.img + (4 * wx) * 28 + 4 * wy;
        if (c1_worker) {
            float patch[8][8];
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const float4 lo = *reinterpret_cast<const float4 *>(ip + r * 28), hi = *reinterpret_cast<const float4 *>(ip + r * 28 + 4);
                patch[r][0] = lo.x; patch[r][1] = lo.y; patch[r][2] = lo.z; patch[r][3] = lo.w;
                patch[r][4] = hi.x; patch[r][5] = hi.y; patch[r][6] = hi.z; patch[r][7] = hi.w;
            }
            float acc[16];
#pragma unroll
            for (int q = 0; q < 16; ++q) acc[q] = 0.0f;
            const float *wc = S.p + L5_C1W + m1 * 25;
#pragma unroll
            for (int i = 0; i < 5; ++i)
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                    const float w = wc[i * 5 + j];
#pragma unroll
                    for (int ox = 0; ox < 4; ++ox)
#pragma unroll
                        for (int oy = 0; oy < 4; ++oy) acc[ox * 4 + oy] = fmaf(w, patch[ox + i][oy + j], acc[ox * 4 + oy]);
                }
            const float bc = S.p[L5_C1B + m1];
            float o[16];
#pragma unroll
            for (int q = 0; q < 16; ++q) o[q] = sigmoid_fast(acc[q] + bc);
#pragma unroll
            for (int ox = 0; ox < 4; ++ox)
                *reinterpret_cast<float4 *>(S.c1o + (m1 * 24 + 4 * wx + ox) * 24 + 4 * wy) = make_float4(o[ox * 4], o[ox * 4 + 1], o[ox * 4 + 2], o[ox * 4 + 3]);
            const float w00 = S.p[L5_S2W], w01 = S.p[L5_S2W + 1], w10 = S.p[L5_S2W + 2], w11 = S.p[L5_S2W + 3], bs = S.p[L5_S2B];
#pragma unroll
            for (int a2 = 0; a2 < 2; ++a2) {
                float v[2];
#pragma unroll
                for (int b2 = 0; b2 < 2; ++b2) {
                    const float sum = w00 * o[(2 * a2) * 4 + 2 * b2] + w01 * o[(2 * a2) * 4 + 2 * b2 + 1] + w10 * o[(2 * a2 + 1) * 4 + 2 * b2] +
                                      w11 * o[(2 * a2 + 1) * 4 + 2 * b2 + 1];
                    v[b2] = sigmoid_fast(sum + bs);
                }
                *reinterpret_cast<float2 *>(S.s2o + (m1 * 12 + 2 * wx + a2) * 12 + 2 * wy) = make_float2(v[0], v[1]);
            }
        }
        __syncthreads();

        // ---- c3: thread (k, x, half) -> outputs y = 4 half .. 4 half + 3; channel order c, i, j
        {
            float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll 2
            for (int c = 0; c < 6; ++c) {
                const float *w = S.p + L5_C3W + (k3 * 6 + c) * 25;
#pragma unroll
                for (int i = 0; i < 5; ++i) {
                    const float *row = S.s2o + (c * 12 + x3 + i) * 12 + 4 * h3;
                    const float4 r0 = *reinterpret_cast<const float4 *>(row), r1 = *reinterpret_cast<const float4 *>(row + 4);
                    const float rr[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
                    for (int j = 0; j < 5; ++j) {
                        const float wv = w[i * 5 + j];
#pragma unroll
                        for (int e = 0; e < 4; ++e) acc[e] = fmaf(wv, rr[e + j], acc[e]);
                    }
                }
            }
            const float bk = S.p[L5_C3B + k3];
            *reinterpret_cast<float4 *>(S.c3o + (k3 * 8 + x3) * 8 + 4 * h3) =
                make_float4(sigmoid_fast(acc[0] + bk), sigmoid_fast(acc[1] + bk), sigmoid_fast(acc[2] + bk), sigmoid_fast(acc[3] + bk));
        }
        __syncthreads();

        // ---- s4 (thread t = output t) and the f layer's partial products
        const float *in4 = S.c3o + (ms * 8 + 2 * xs) * 8 + 2 * ys;
        const float2 i0 = *reinterpret_cast<const float2 *>(in4), i1 = *reinterpret_cast<const float2 *>(in4 + 8);
        const float s4v = sigmoid_fast(S.p[L5_S4W] * i0.x + S.p[L5_S4W + 1] * i0.y + S.p[L5_S4W + 2] * i1.x + S.p[L5_S4W + 3] * i1.y + S.p[L5_S4B]);
        float fw[10], fcp[16];
#pragma unroll
        for (int q = 0; q < 16; ++q) fcp[q] = 0.0f;
#pragma unroll
        for (int q = 0; q < 10; ++q) {
            fw[q] = S.p[L5_FW + q * 256 + t];
            fcp[q] = fw[q] * s4v;
        }
        {
            const float v = warp_sum16_transposed(fcp, lane);                // lane 2q (and 2q + 1) holds output q's warp sum
            if ((lane & 1) == 0 && (lane >> 1) < 10) S.fc_red[warp][lane >> 1] = v;
        }
        __syncthreads();
        // f output (layer.h:184-211), makeError (layer.h:91-95): every warp for itself
        float d = 0.0f;
        if (lane < 10) {
            float pre = 0.0f;
#pragma unroll
            for (int w = 0; w < 8; ++w) pre += S.fc_red[w][lane];
            const float out = sigmoid_fast(pre + S.p[L5_FB + lane]);
            if (warp == 0) S.fo[lane] = out;
            d = (lane == label ? 1.0f : 0.0f) - out;
        }
        if (!TRAIN) {
            __syncthreads();
            if (t < 10 && a.f_out) a.f_out[(size_t)b * 10 + t] = S.fo[t];
            continue;
        }
        float dq[10];
#pragma unroll
        for (int q = 0; q < 10; ++q) dq[q] = __shfl_sync(0xffffffffu, d, q);
        if (warp == 0) {
            gfb += d;                                                        // lanes 0..9: the f bias entries
            float ss = 0.0f;
#pragma unroll
            for (int q = 0; q < 10; ++q) ss = fmaf(dq[q], dq[q], ss);
            err_acc += sqrtf(ss);                                            // vectorNorm, Main.cpp:28-34 (lane 0's copy is reported)
        }
        // ---- backward: f and s4 are thread-local
        float dps4;
        {
            float dout = 0.0f;
#pragma unroll
            for (int q = 0; q < 10; ++q) {
                gfw[q] = fmaf(dq[q], s4v, gfw[q]);                           // rule of bp_weight_f, layer.h:214-227
                dout = fmaf(fw[q], dq[q], dout);                             // rule of bp_output_s1, layer.h:237-257
            }
            dps4 = dout * s4v * (1.0f - s4v);                                // rule of bp_preact_s1, layer.h:260-270
            S.dpre_s4[t] = dps4;
            // s4 weight / bias gradient (rule of bp_weight_s1 / bp_bias_s1, layer.h:272-314): 5 block sums
            const float pr[5] = {dps4 * i0.x, dps4 * i0.y, dps4 * i1.x, dps4 * i1.y, dps4};
#pragma unroll
            for (int e = 0; e < 5; ++e) {
                const float v = warp_sum(pr[e]);
                if (lane == 0) S.part[warp][e] = v;
            }
        }
        __syncthreads();
        if (t < 5) {
            float v = 0.0f;
#pragma unroll
            for (int w = 0; w < 8; ++w) v += S.part[w][t];
            S.gacc[L5_S4W + t] += v;                                         // t == 4 lands on L5_S4B
        }
        // ---- d_preact of c3 (rule of bp_output_c1 + bp_preact_c1, layer.h:319-369) into the padded array; c3 bias sums
        {
            const float2 dd = *reinterpret_cast<const float2 *>(S.dpre_s4 + (k3 * 4 + (x3 >> 1)) * 4 + 2 * h3);
            const float4 ov = *reinterpret_cast<const float4 *>(S.c3o + (k3 * 8 + x3) * 8 + 4 * h3);
            const float wa = S.p[L5_S4W + (x3 & 1) * 2], wb = S.p[L5_S4W + (x3 & 1) * 2 + 1];
            float4 dp;
            dp.x = wa * dd.x * (ov.x * (1.0f - ov.x));
            dp.y = wb * dd.x * (ov.y * (1.0f - ov.y));
            dp.z = wa * dd.y * (ov.z * (1.0f - ov.z));
            dp.w = wb * dd.y * (ov.w * (1.0f - ov.w));
            *reinterpret_cast<float4 *>(S.dpad + (k3 * 16 + x3 + 4) * 16 + 4 * h3 + 4) = dp;
            float sb = (dp.x + dp.y) + (dp.z + dp.w);
            sb += __shfl_xor_sync(0xffffffffu, sb, 8);
            sb += __shfl_xor_sync(0xffffffffu, sb, 4);
            sb += __shfl_xor_sync(0xffffffffu, sb, 2);
            sb += __shfl_xor_sync(0xffffffffu, sb, 1);
            if ((lane & 15) == 0) S.gacc[L5_C3B + k3] += sb;
        }
        __syncthreads();
        // ---- c3 weight gradient: item (k, c, i) = 5 taps x 64 products, /64 as they are added (layer.h:389 by rule)
        for (int it = t; it < 480; it += L5_T) {
            const int k = it / 30, c = (it / 5) % 6, i = it % 5;
            float sj[5] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
            for (int x = 0; x < 8; ++x) {
                const float *dr = S.dpad + (k * 16 + x + 4) * 16 + 4;
                const float4 d0 = *reinterpret_cast<const float4 *>(dr), d1 = *reinterpret_cast<const float4 *>(dr + 4);
                const float *sr = S.s2o + (c * 12 + x + i) * 12;
                const float4 s0 = *reinterpret_cast<const float4 *>(sr), s1 = *reinterpret_cast<const float4 *>(sr + 4),
                             s2 = *reinterpret_cast<const float4 *>(sr + 8);
                const float dv[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
                const float sv[12] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w, s2.x, s2.y, s2.z, s2.w};
#pragma unroll
                for (int j = 0; j < 5; ++j)
#pragma unroll
                    for (int y = 0; y < 8; ++y) sj[j] = fmaf(dv[y], sv[y + j], sj[j]);
            }
            float *g = S.gacc + L5_C3W + (k * 6 + c) * 25 + i * 5;
#pragma unroll
            for (int j = 0; j < 5; ++j) g[j] += sj[j] * (1.0f / 64.0f);
        }
        // ---- d_preact of s2: the adjoint of c3 (no counterpart in the reference) over the zero-padded array, 4 outputs per thread
        float ps[5] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
        if (c1_worker) {
            float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll 2
            for (int k = 0; k < 16; ++k) {
                const float *w = S.p + L5_C3W + (k * 6 + c2) * 25;
#pragma unroll
                for (int i = 0; i < 5; ++i) {
                    const float *row = S.dpad + (k * 16 + u2 + 4 - i) * 16 + 4 * g2;
                    const float4 r0 = *reinterpret_cast<const float4 *>(row), r1 = *reinterpret_cast<const float4 *>(row + 4);
                    const float rr[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
                    for (int j = 0; j < 5; ++j) {
                        const float wv = w[i * 5 + j];
#pragma unroll
                        for (int e = 0; e < 4; ++e) acc[e] = fmaf(wv, rr[e + 4 - j], acc[e]);
                    }
                }
            }
            const float4 ov = *reinterpret_cast<const float4 *>(S.s2o + (c2 * 12 + u2) * 12 + 4 * g2);
            const float dp[4] = {acc[0] * ov.x * (1.0f - ov.x), acc[1] * ov.y * (1.0f - ov.y), acc[2] * ov.z * (1.0f - ov.z),
                                 acc[3] * ov.w * (1.0f - ov.w)};
            *reinterpret_cast<float4 *>(S.dpre_s2 + (c2 * 12 + u2) * 12 + 4 * g2) = make_float4(dp[0], dp[1], dp[2], dp[3]);
            // s2 weight / bias gradient partials: products with the c1 outputs under this thread's 4 pooled positions
#pragma unroll
            for (int a2 = 0; a2 < 2; ++a2) {
                const float *cr = S.c1o + (c2 * 24 + 2 * u2 + a2) * 24 + 8 * g2;
                const float4 q0 = *reinterpret_cast<const float4 *>(cr), q1 = *reinterpret_cast<const float4 *>(cr + 4);
                const float cv[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    ps[a2 * 2] = fmaf(dp[e], cv[2 * e], ps[a2 * 2]);
                    ps[a2 * 2 + 1] = fmaf(dp[e], cv[2 * e + 1], ps[a2 * 2 + 1]);
                }
            }
            ps[4] = (dp[0] + dp[1]) + (dp[2] + dp[3]);
        }
#pragma unroll
        for (int e = 0; e < 5; ++e) {
            const float v = warp_sum(ps[e]);
            if (lane == 0) S.part[warp][e] = v;
        }
        __syncthreads();
        if (t < 5) {
            float v = 0.0f;
#pragma unroll
            for (int w = 0; w < 8; ++w) v += S.part[w][t];
            S.gacc[L5_S2W + t] += v;                                         // t == 4 lands on L5_S2B
        }
        // ---- d_preact of c1 for this thread's window, c1 weight-gradient partials (bp_weight_c1 / bp_bias_c1, layer.h:371-410)
        if (c1_worker) {
            float dpc[16];
            float bsum = 0.0f;
            const float sw[4] = {S.p[L5_S2W], S.p[L5_S2W + 1], S.p[L5_S2W + 2], S.p[L5_S2W + 3]};
#pragma unroll
            for (int ox = 0; ox < 4; ++ox) {
                const float4 ov = *reinterpret_cast<const float4 *>(S.c1o + (m1 * 24 + 4 * wx + ox) * 24 + 4 * wy);
                const float2 dd = *reinterpret_cast<const float2 *>(S.dpre_s2 + (m1 * 12 + 2 * wx + (ox >> 1)) * 12 + 2 * wy);
                const float o4[4] = {ov.x, ov.y, ov.z, ov.w};
#pragma unroll
                for (int oy = 0; oy < 4; ++oy) {
                    const float dout = sw[(ox & 1) * 2 + (oy & 1)] * (oy < 2 ? dd.x : dd.y);
                    dpc[ox * 4 + oy] = dout * (o4[oy] * (1.0f - o4[oy]));
                    bsum += dpc[ox * 4 + oy];
                }
            }
            float patch[8][8];
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const float4 lo = *reinterpret_cast<const float4 *>(ip + r * 28), hi = *reinterpret_cast<const float4 *>(ip + r * 28 + 4);
                patch[r][0] = lo.x; patch[r][1] = lo.y; patch[r][2] = lo.z; patch[r][3] = lo.w;
                patch[r][4] = hi.x; patch[r][5] = hi.y; patch[r][6] = hi.z; patch[r][7] = hi.w;
            }
            float *row = S.red + t * 27;
#pragma unroll
            for (int i = 0; i < 5; ++i)
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                    float sacc = 0.0f;
#pragma unroll
                    for (int ox = 0; ox < 4; ++ox)
#pragma unroll
                        for (int oy = 0; oy < 4; ++oy) sacc = fmaf(dpc[ox * 4 + oy], patch[ox + i][oy + j], sacc);
                    row[i * 5 + j] = sacc;
                }
            row[25] = bsum;
        }
        __syncthreads();
        if (t < 156) {                       // 150 c1 taps + 6 c1 bias sums over the 36 windows of a map
            const int mm = t < 150 ? t / 25 : t - 150;
            const int col = t < 150 ? t % 25 : 25;
            const float *r = S.red + (mm * 36) * 27 + col;
            float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
#pragma unroll
            for (int w = 0; w < 36; w += 4) {
                s0 += r[(w + 0) * 27];
                s1 += r[(w + 1) * 27];
                s2 += r[(w + 2) * 27];
                s3 += r[(w + 3) * 27];
            }
            const float ssum = (s0 + s1) + (s2 + s3);
            if (t < 150) S.gacc[L5_C1W + t] += ssum * (1.0f / 576.0f);
            else S.gacc[L5_C1B + mm] += ssum;
        }
    }
    if (TRAIN) {
        __syncthreads();
        float *slot = a.slots + (size_t)blockIdx.x * L5_NPK;
        for (int j = t; j < L5_FW; j += L5_T) slot[j] = S.gacc[j];
#pragma unroll
        for (int q = 0; q < 10; ++q) slot[L5_FW + q * 256 + t] = gfw[q];
        if (t < 10) slot[L5_FB + t] = gfb;
        if (t == 0) slot[L5_NP] = err_acc;
    }
}

// fixed-order sum of the per-CTA slots; update = 1: w += step * g with the bias divisors of the rules (layer.h:99, 316, 412)
__global__ void __launch_bounds__(256) k_l5_reduce(const float *slots, int nslots, float *grads, float *params, float step, int update) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > L5_NP) return;
    float g = 0.0f;
    for (int k = 0; k < nslots; ++k) g += slots[(size_t)k * L5_NPK + j];
    if (grads) grads[j] = g;
    if (update && j < L5_NP) {
        float d = step * g;
        if (j >= L5_C1B && j < L5_S2W) d = d / 576.0f;
        else if (j == L5_S2B) d = d / 864.0f;
        else if (j >= L5_C3B && j < L5_S4W) d = d / 64.0f;
        else if (j == L5_S4B) d = d / 256.0f;
        params[j] += d;
    }
}

int l5_grid(pcnn_ctx *ctx, int B) {
    const int cap = ctx->sm_count * 2;
    return B < cap ? B : cap;
}

template <bool TRAIN> int l5_launch(pcnn_ctx *ctx, const L5Args &a, int grid) {
    static bool configured[2][64] = {};
    if (!configured[TRAIN][ctx->device & 63]) {
        PCNN_CUDA(cudaFuncSetAttribute(k_l5_step<TRAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(L5Smem)));
        configured[TRAIN][ctx->device & 63] = true;
    }
    k_l5_step<TRAIN><<<grid, L5_T, sizeof(L5Smem), ctx->stream>>>(a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

int l5_grads(pcnn_ctx *ctx, float *params_dev, const void *images, int pixel_type, const uint8_t *labels, int B, float *grads_dev,
             int update) {
    PCNN_REQUIRE(ctx && params_dev && images && labels && B > 0, PCNN_ERR_ARG, "pcnn_l5: NULL argument or B <= 0");
    PCNN_REQUIRE(pixel_type == PCNN_U8 || pixel_type == PCNN_F32, PCNN_ERR_ARG, "pcnn_l5: bad pixel type %d", pixel_type);
    pcnn_device_guard g(ctx->device);
    const int grid = l5_grid(ctx, B);
    float *slots = nullptr;
    int rc = pcnn_scratch(ctx, (size_t)grid * L5_NPK * sizeof(float), (void **)&slots);
    if (rc) return rc;
    L5Args a{};
    a.images = images; a.labels = labels; a.params = params_dev; a.slots = slots; a.B = B; a.pixel_u8 = pixel_type == PCNN_U8;
    if ((rc = l5_launch<true>(ctx, a, grid))) return rc;
    k_l5_reduce<<<(L5_NP + 1 + 255) / 256, 256, 0, ctx->stream>>>(slots, grid, grads_dev, params_dev, ctx->lr / (float)B, update);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

}  // namespace

extern "C" int pcnn_l5_compute_grads(pcnn_ctx *ctx, const float *params_dev, const void *images_dev, int pixel_type,
                                     const uint8_t *labels_dev, int B, float *grads_dev) {
    PCNN_REQUIRE(grads_dev, PCNN_ERR_ARG, "pcnn_l5_compute_grads: NULL output");
    return l5_grads(ctx, const_cast<float *>(params_dev), images_dev, pixel_type, labels_dev, B, grads_dev, 0);
}

extern "C" int pcnn_l5_train_step(pcnn_ctx *ctx, float *params_dev, const void *images_dev, int pixel_type, const uint8_t *labels_dev,
                                  int B, float *grads_dev) {
    return l5_grads(ctx, params_dev, images_dev, pixel_type, labels_dev, B, grads_dev, 1);
}

extern "C" int pcnn_l5_forward(pcnn_ctx *ctx, const float *params_dev, const void *images_dev, int pixel_type, int B, float *f_out_dev) {
    PCNN_REQUIRE(ctx && params_dev && images_dev && f_out_dev && B > 0, PCNN_ERR_ARG, "pcnn_l5_forward: NULL argument or B <= 0");
    PCNN_REQUIRE(pixel_type == PCNN_U8 || pixel_type == PCNN_F32, PCNN_ERR_ARG, "pcnn_l5_forward: bad pixel type %d", pixel_type);
    pcnn_device_guard g(ctx->device);
    L5Args a{};
    a.images = images_dev; a.params = params_dev; a.f_out = f_out_dev; a.B = B; a.pixel_u8 = pixel_type == PCNN_U8;
    return l5_launch<false>(ctx, a, l5_grid(ctx, B));
}
