// parallel-cnn_b200/csrc/batchnorm_nhwc.cu -- batch normalization of the dense bf16 NHWC [pixels][C] activations the conv
// forwards write (pcnn_batchnorm_nhwc_bf16_fwd / _bwd), with the residual add and the ReLU of a ResNet block fused into the
// elementwise pass, or SiLU, hard-swish or ReLU6, whose backward (pcnn_batchnorm_nhwc_bf16_bwd_preact) takes the derivative at the
// pre-activation recomputed from x, beta and r instead of from y.  The contract, every operation in its order, is in include/pcnn.h.
//
// The passes at codes 0, 3 and 6 are HBM-bound; those at 4 (SiLU) and 5 (hard-swish) are bound by instruction issue (the
// exponential and the quotients per element).  With C % 8 == 0 a thread moves 16-byte vectors of 8 channels of one pixel, otherwise single
// elements.  All passes share one partition: CTA b owns the pixels [b * BN_ITERS * lanes, (b + 1) * BN_ITERS * lanes), thread
// t keeps channel group g = t % G (G = C / VEC groups, lanes = 256 / G) of the pixels lane, lane + lanes, ... (lane = t / G), so
// consecutive threads touch consecutive bytes.  A thread loads bn_unroll pixels before it uses any (in place, dx == dy, each
// element is read and then written by the same thread).
//
// Forward, training: k_bn_stats sums d = x - k and d * d per channel in fp32, k being the CTA's first pixel (a shift taken from
// the data, so the sums do not cancel when the mean is large next to the spread), thread by thread, then lane by lane in lane
// order into the CTA's slot {k, sum d, sum d^2}.  k_bn_finalize merges the slots in double in a fixed order: the mean from
// sum n_b k_b + s1_b, then M2 = sum (s2_b - s1_b^2 / n_b) + n_b (mean_b - mean)^2 (Chan's formula in two passes).  k_bn_apply
// then reads x a second time.  Backward: k_bn_bwd_reduce sums g~ and g~ * xhat into per-CTA slots that
// pcnn_conv_wgrad_reduce_slots adds in a fixed order into dbeta and dgamma; k_bn_bwd_dx reads them back.  Nothing depends on the
// SM count and there are no atomics: the bits are the same on every run and every H100.
#include "pcnn_internal.h"
#include "tc_common.cuh"

#include <cuda_bf16.h>

#include <math.h>

namespace {

constexpr int BN_THREADS = 256;
constexpr int BN_ITERS = 16;         // pixels per thread
constexpr int BN_MIN_CTAS = 2;       // CTAs per SM the register budget leaves room for
constexpr int BN_MAX_C = 256;

#include "norm_act.cuh"

// per-CTA sums of the lanes of two [lanes][C] planes in lane order -> slots[plane][cta][C]
__device__ __forceinline__ void bn_cta_sums(const float *part, int lanes, int C, float *slots, long ctas) {
    for (int t = threadIdx.x; t < 2 * C; t += BN_THREADS) {
        const int which = t / C, c = t - which * C;
        const float *p = part + which * BN_THREADS * 8;
        float s = 0.0f;
        for (int l = 0; l < lanes; ++l) s = __fadd_rn(s, p[l * C + c]);
        slots[((long)which * ctas + blockIdx.x) * C + c] = s;
    }
}

template <int VEC>
__global__ void __launch_bounds__(BN_THREADS, BN_MIN_CTAS) k_bn_stats(const __nv_bfloat16 *__restrict__ x, float *__restrict__ slots, long pixels, int C,
                                                         long ctas) {
    __shared__ float part[2 * BN_THREADS * 8];        // two [lanes][C] planes: lanes * C <= 256 * VEC
    constexpr int U = bn_unroll<VEC>();
    const int G = C / VEC, lanes = BN_THREADS / G;
    const int lane = threadIdx.x / G, g = threadIdx.x % G;
    const long p0 = (long)blockIdx.x * BN_ITERS * lanes;
    if (lane < lanes) {
        const BfVec<VEC> kv = ld<VEC>(x + p0 * C + g * VEC);     // the CTA's first pixel: every thread's shift
        float k[VEC], s1[VEC], s2[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
            k[i] = __bfloat162float(kv.h[i]);
            s1[i] = s2[i] = 0.0f;
        }
        for (int j0 = 0; j0 < BN_ITERS; j0 += U) {
            BfVec<VEC> v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long px = p0 + lane + (long)(j0 + u) * lanes;
                if (px < pixels) v[u] = ld<VEC>(x + px * C + g * VEC);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (p0 + lane + (long)(j0 + u) * lanes >= pixels) continue;
#pragma unroll
                for (int i = 0; i < VEC; ++i) {
                    const float d = __fsub_rn(__bfloat162float(v[u].h[i]), k[i]);
                    s1[i] = __fadd_rn(s1[i], d);
                    s2[i] = __fadd_rn(s2[i], __fmul_rn(d, d));
                }
            }
        }
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
            part[lane * C + g * VEC + i] = s1[i];
            part[BN_THREADS * 8 + lane * C + g * VEC + i] = s2[i];
        }
    }
    __syncthreads();
    bn_cta_sums(part, lanes, C, slots + ctas * C, ctas);          // planes 1 and 2: sum d, sum d^2
    for (int c = threadIdx.x; c < C; c += BN_THREADS) slots[(long)blockIdx.x * C + c] = __bfloat162float(x[p0 * C + c]);   // plane 0: k
}

// one CTA of 32 x 32 threads per 32 channels: thread (cx, sy) merges the slots sy, sy + 32, ... of channel 32 blockIdx.x + cx in
// double, then the 32 partials are added in a fixed pairwise tree (a handful of CTAs walking the slots one by one would take
// longer than the statistics pass)
constexpr int FIN_ROWS = 32;

__device__ __forceinline__ double bn_tree(double (*part)[33], int cx, int sy, double v) {
    part[sy][cx] = v;
    __syncthreads();
    for (int s = FIN_ROWS / 2; s >= 1; s /= 2) {
        if (sy < s) part[sy][cx] += part[sy + s][cx];
        __syncthreads();
    }
    const double out = part[0][cx];
    __syncthreads();                                  // part is reused
    return out;
}

__global__ void __launch_bounds__(32 * FIN_ROWS) k_bn_finalize(const float *__restrict__ slots, long ctas, long pixels, int C, long per_cta,
                                                               float eps, float momentum, float *save_mean, float *save_rstd, float *run_mean,
                                                               float *run_var) {
    __shared__ double part[FIN_ROWS][33];
    const int cx = threadIdx.x & 31, sy = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + cx;
    const bool on = c < C;
    const float *K = slots, *S1 = slots + ctas * C, *S2 = slots + 2 * ctas * C;
    double a = 0.0;
    if (on)
#pragma unroll 4
        for (long b = sy; b < ctas; b += FIN_ROWS) {
            const double n = (double)min(per_cta, pixels - b * per_cta);
            a += n * (double)K[b * C + c] + (double)S1[b * C + c];
        }
    const double M = (double)pixels;
    const double mean = bn_tree(part, cx, sy, a) / M;
    a = 0.0;
    if (on)
#pragma unroll 4
        for (long b = sy; b < ctas; b += FIN_ROWS) {
            const double n = (double)min(per_cta, pixels - b * per_cta);
            const double s1 = (double)S1[b * C + c];
            const double d = ((double)K[b * C + c] + s1 / n) - mean;
            a += ((double)S2[b * C + c] - s1 * (s1 / n)) + n * d * d;
        }
    const double m2 = fmax(bn_tree(part, cx, sy, a), 0.0);
    if (sy != 0 || !on) return;
    save_mean[c] = (float)mean;
    save_rstd[c] = (float)__drcp_rn(__dsqrt_rn(m2 / M + (double)eps));
    if (run_mean) {
        const float keep = __fsub_rn(1.0f, momentum);
        run_mean[c] = __fadd_rn(__fmul_rn(keep, run_mean[c]), __fmul_rn(momentum, (float)mean));
        run_var[c] = __fadd_rn(__fmul_rn(keep, run_var[c]), __fmul_rn(momentum, (float)(m2 / (M - 1.0))));
    }
}

// y = bf16_rn(act(xhat * gamma + beta (+ float(r)))); mean and rstd from the saved statistics (training) or mean = running_mean
// and rstd = float(1 / sqrt(double(running_var) + eps)) (eval, var != nullptr)
template <int VEC, int ACT>
__global__ void __launch_bounds__(BN_THREADS, BN_MIN_CTAS) k_bn_apply(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ r,
                                                         __nv_bfloat16 *__restrict__ y, const float *__restrict__ mean,
                                                         const float *__restrict__ rstd, const float *__restrict__ var, float eps,
                                                         const float *__restrict__ gamma, const float *__restrict__ beta, long pixels, int C) {
    constexpr int U = bn_unroll<VEC>();
    const int G = C / VEC, lanes = BN_THREADS / G;
    const int lane = threadIdx.x / G, g = threadIdx.x % G;
    if (lane >= lanes) return;
    float mu[VEC], rs[VEC], ga[VEC], be[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        const int c = g * VEC + i;
        mu[i] = mean[c];
        rs[i] = var ? (float)__drcp_rn(__dsqrt_rn((double)var[c] + (double)eps)) : rstd[c];
        ga[i] = gamma[c];
        be[i] = beta[c];
    }
    const long p0 = (long)blockIdx.x * BN_ITERS * lanes + lane;
    for (int j0 = 0; j0 < BN_ITERS; j0 += U) {
        BfVec<VEC> xv[U], rv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long px = p0 + (long)(j0 + u) * lanes;
            if (px < pixels) {
                xv[u] = ld<VEC>(x + px * C + g * VEC);
                if (r) rv[u] = ld<VEC>(r + px * C + g * VEC);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long px = p0 + (long)(j0 + u) * lanes;
            if (px >= pixels) continue;
            BfVec<VEC> out;
#pragma unroll
            for (int i = 0; i < VEC; ++i) {
                float v = __fadd_rn(__fmul_rn(bn_xhat(xv[u].h[i], mu[i], rs[i]), ga[i]), be[i]);
                if (r) v = __fadd_rn(v, __bfloat162float(rv[u].h[i]));
                out.h[i] = __float2bfloat16_rn(bn_act_f32<ACT>(v));
            }
            st<VEC>(y + px * C + g * VEC, out);
        }
    }
}

// first backward pass: per-CTA slots [0][cta][C] = sum g~, [1][cta][C] = sum g~ * xhat.  At codes 4-6 g~ comes from the
// pre-activation recomputed from x, beta and r (y is not read); their per-channel constants live in shared memory.
template <int VEC, int ACT>
__global__ void __launch_bounds__(BN_THREADS, BN_MIN_CTAS) k_bn_bwd_reduce(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ y,
                                                              const __nv_bfloat16 *__restrict__ r, const __nv_bfloat16 *__restrict__ dy,
                                                              const __nv_bfloat16 *__restrict__ dy2, const float *__restrict__ mean,
                                                              const float *__restrict__ rstd, const float *__restrict__ gamma,
                                                              const float *__restrict__ beta, float *__restrict__ slots, long pixels, int C,
                                                              long ctas) {
    constexpr bool PRE = bn_preact<ACT>();
    __shared__ float part[2 * BN_THREADS * 8];
    __shared__ float cmu[PRE ? BN_MAX_C : 1], crs[PRE ? BN_MAX_C : 1], cga[PRE ? BN_MAX_C : 1], cbe[PRE ? BN_MAX_C : 1];
    constexpr int U = bn_unroll<VEC>();
    const int G = C / VEC, lanes = BN_THREADS / G;
    const int lane = threadIdx.x / G, g = threadIdx.x % G;
    if (PRE) {
        for (int c = threadIdx.x; c < C; c += BN_THREADS) {
            cmu[c] = mean[c];
            crs[c] = rstd[c];
            cga[c] = gamma[c];
            cbe[c] = beta[c];
        }
        __syncthreads();
    }
    if (lane < lanes) {
        float mu[PRE ? 1 : VEC], rs[PRE ? 1 : VEC], sb[VEC], sg[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
            if (!PRE) {
                mu[i] = mean[g * VEC + i];
                rs[i] = rstd[g * VEC + i];
            }
            sb[i] = sg[i] = 0.0f;
        }
        const long p0 = (long)blockIdx.x * BN_ITERS * lanes + lane;
        for (int j0 = 0; j0 < BN_ITERS; j0 += U) {
            BfVec<VEC> xv[U], yv[U], dv[U], d2[U], rv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long px = p0 + (long)(j0 + u) * lanes;
                if (px < pixels) {
                    const long off = px * C + g * VEC;
                    xv[u] = ld<VEC>(x + off);
                    dv[u] = ld<VEC>(dy + off);
                    if (ACT == PCNN_ACT_RELU) yv[u] = ld<VEC>(y + off);
                    if (PRE && r) rv[u] = ld<VEC>(r + off);
                    if (dy2) d2[u] = ld<VEC>(dy2 + off);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (p0 + (long)(j0 + u) * lanes >= pixels) continue;
#pragma unroll
                for (int i = 0; i < VEC; ++i) {
                    if constexpr (PRE) {
                        const int c = g * VEC + i;
                        const float xh = bn_xhat(xv[u].h[i], cmu[c], crs[c]);
                        const float gt =
                            __bfloat162float(bn_dgrad_pre<ACT>(dv[u].h[i], d2[u].h[i], dy2 != nullptr, bn_pre(xh, cga[c], cbe[c], r, rv[u].h[i])));
                        sb[i] = __fadd_rn(sb[i], gt);
                        sg[i] = __fadd_rn(sg[i], __fmul_rn(gt, xh));
                    } else {
                        const float gt = __bfloat162float(bn_dgrad<ACT>(dv[u].h[i], d2[u].h[i], dy2 != nullptr, yv[u].h[i]));
                        sb[i] = __fadd_rn(sb[i], gt);
                        sg[i] = __fadd_rn(sg[i], __fmul_rn(gt, bn_xhat(xv[u].h[i], mu[i], rs[i])));
                    }
                }
            }
        }
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
            part[lane * C + g * VEC + i] = sb[i];
            part[BN_THREADS * 8 + lane * C + g * VEC + i] = sg[i];
        }
    }
    __syncthreads();
    bn_cta_sums(part, lanes, C, slots, ctas);
}

// second backward pass: dx = bf16_rn(((g~ - dbeta / M) - xhat * (dgamma / M)) * (gamma * rstd)), dr = g~.  dx may be dy.
template <int VEC, int ACT>
__global__ void __launch_bounds__(BN_THREADS, BN_MIN_CTAS) k_bn_bwd_dx(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ y,
                                                          const __nv_bfloat16 *__restrict__ r, const __nv_bfloat16 *dy,
                                                          const __nv_bfloat16 *__restrict__ dy2, const float *__restrict__ mean,
                                                          const float *__restrict__ rstd, const float *__restrict__ gamma,
                                                          const float *__restrict__ beta, const float *__restrict__ dgamma,
                                                          const float *__restrict__ dbeta, __nv_bfloat16 *dx, __nv_bfloat16 *__restrict__ dr,
                                                          long pixels, int C, float Mf) {
    constexpr bool PRE = bn_preact<ACT>();
    constexpr int U = bn_unroll<VEC>();
    const int G = C / VEC, lanes = BN_THREADS / G;
    const int lane = threadIdx.x / G, g = threadIdx.x % G;
    // the per-channel constants live in shared memory: forty of them in registers next to the loads spill on the 8-channel path
    __shared__ float mu[BN_MAX_C], rs[BN_MAX_C], mb[BN_MAX_C], mg[BN_MAX_C], sc[BN_MAX_C];
    __shared__ float ga[PRE ? BN_MAX_C : 1], be[PRE ? BN_MAX_C : 1];
    for (int c = threadIdx.x; c < C; c += BN_THREADS) {
        mu[c] = mean[c];
        rs[c] = rstd[c];
        mb[c] = __fdiv_rn(dbeta[c], Mf);
        mg[c] = __fdiv_rn(dgamma[c], Mf);
        sc[c] = __fmul_rn(gamma[c], rs[c]);
        if (PRE) {
            ga[c] = gamma[c];
            be[c] = beta[c];
        }
    }
    __syncthreads();
    if (lane >= lanes) return;
    const long p0 = (long)blockIdx.x * BN_ITERS * lanes + lane;
    for (int j0 = 0; j0 < BN_ITERS; j0 += U) {
        BfVec<VEC> xv[U], yv[U], dv[U], d2[U], rv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long px = p0 + (long)(j0 + u) * lanes;
            if (px < pixels) {
                const long off = px * C + g * VEC;
                xv[u] = ld<VEC>(x + off);
                dv[u] = ld<VEC>(dy + off);
                if (ACT == PCNN_ACT_RELU) yv[u] = ld<VEC>(y + off);
                if (PRE && r) rv[u] = ld<VEC>(r + off);
                if (dy2) d2[u] = ld<VEC>(dy2 + off);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long px = p0 + (long)(j0 + u) * lanes;
            if (px >= pixels) continue;
            BfVec<VEC> o, gv;
#pragma unroll
            for (int i = 0; i < VEC; ++i) {
                const int c = g * VEC + i;
                const float xh = bn_xhat(xv[u].h[i], mu[c], rs[c]);
                if constexpr (PRE)
                    gv.h[i] = bn_dgrad_pre<ACT>(dv[u].h[i], d2[u].h[i], dy2 != nullptr, bn_pre(xh, ga[c], be[c], r, rv[u].h[i]));
                else
                    gv.h[i] = bn_dgrad<ACT>(dv[u].h[i], d2[u].h[i], dy2 != nullptr, yv[u].h[i]);
                const float t = __fsub_rn(__fsub_rn(__bfloat162float(gv.h[i]), mb[c]), __fmul_rn(xh, mg[c]));
                o.h[i] = __float2bfloat16_rn(__fmul_rn(t, sc[c]));
            }
            const long off = px * C + g * VEC;
            st<VEC>(dx + off, o);
            if (dr) st<VEC>(dr + off, gv);
        }
    }
}

struct BnGeom {
    int vec, lanes;
    long per_cta, ctas;
};

// the shape rules of pcnn.h, refused with PCNN_ERR_ARG and a message naming `fn`
int bn_geom(const char *fn, long pixels, int C, int training, BnGeom *out) {
    PCNN_REQUIRE(training == 0 || training == 1, PCNN_ERR_ARG, "%s: training = %d: 0 (eval) or 1 (training) is required", fn, training);
    PCNN_REQUIRE(C >= 1 && C <= BN_MAX_C, PCNN_ERR_ARG, "%s: C = %d channels: 1 <= C <= 256 is required", fn, C);
    if (training)
        PCNN_REQUIRE(pixels >= 2, PCNN_ERR_ARG,
                     "%s: pixels = %ld: training needs more than 1 value per channel (pixels = N * H * W >= 2)", fn, pixels);
    else
        PCNN_REQUIRE(pixels >= 1, PCNN_ERR_ARG, "%s: pixels = %ld: at least one pixel (N * H * W) is required", fn, pixels);
    out->vec = C % 8 == 0 ? 8 : 1;
    out->lanes = BN_THREADS / (C / out->vec);
    out->per_cta = (long)BN_ITERS * out->lanes;
    out->ctas = (pixels + out->per_cta - 1) / out->per_cta;
    PCNN_REQUIRE(out->ctas < (1L << 31), PCNN_ERR_ARG, "%s: %ld pixels exceed the grid", fn, pixels);
    return PCNN_OK;
}

enum BnPass { BN_FWD, BN_BWD, BN_BWD_PREACT };

bool act_from_preact(int act) { return act == PCNN_ACT_SILU || act == PCNN_ACT_HARDSWISH || act == PCNN_ACT_RELU6; }

// the codes each entry takes: the forward 0 and 3-6, the backward 0 and 3, the pre-activation backward 4-6
int bn_act(const char *fn, int act, BnPass pass) {
    PCNN_REQUIRE(act != PCNN_ACT_SIGMOID, PCNN_ERR_ARG,
                 "%s: act 1 (sigmoid) is not available after batch normalization: sigmoid_bf16 uses tanh.approx, which no reference "
                 "can replay bit for bit; %s is required", fn,
                 pass == BN_BWD_PREACT ? "act 4 (SiLU), 5 (hard-swish) or 6 (ReLU6)" : "act 0 (none) or 3 (ReLU)");
    const bool plain = act == PCNN_ACT_NONE || act == PCNN_ACT_RELU, pre = act_from_preact(act);
    if (pass == BN_FWD)
        PCNN_REQUIRE(plain || pre, PCNN_ERR_ARG, "%s: act %d is not 0 (none) or 3 (ReLU), nor 4 (SiLU), 5 (hard-swish) or 6 (ReLU6)", fn, act);
    if (pass == BN_BWD) {
        PCNN_REQUIRE(!pre, PCNN_ERR_ARG,
                     "%s: act %d takes its gradient from the recomputed pre-activation, not from y: pcnn_batchnorm_nhwc_bf16_bwd_preact "
                     "is its backward", fn, act);
        PCNN_REQUIRE(plain, PCNN_ERR_ARG, "%s: act %d is not 0 (none) or 3 (ReLU)", fn, act);
    }
    if (pass == BN_BWD_PREACT) {
        PCNN_REQUIRE(!plain, PCNN_ERR_ARG, "%s: act %d takes its gradient from y: pcnn_batchnorm_nhwc_bf16_bwd is its backward", fn, act);
        PCNN_REQUIRE(pre, PCNN_ERR_ARG, "%s: act %d is not 4 (SiLU), 5 (hard-swish) or 6 (ReLU6)", fn, act);
    }
    return PCNN_OK;
}

// column of an accepted code in the kernel tables: 0, 3, 4, 5, 6 -> 0 .. 4
int act_col(int act) { return act == PCNN_ACT_NONE ? 0 : act - 2; }

struct Buf {
    const void *p;
    size_t n;
};

bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// true when no two of the non-NULL buffers share a byte, except a and b when they are the same buffer (in place)
bool disjoint(const Buf *b, int n, const void *same_a = nullptr, const void *same_b = nullptr) {
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

typedef void (*apply_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, __nv_bfloat16 *, const float *, const float *, const float *, float,
                         const float *, const float *, long, int);
typedef void (*reduce_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *,
                          const float *, const float *, const float *, const float *, float *, long, int, long);
typedef void (*dx_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *,
                      const float *, const float *, const float *, const float *, const float *, const float *, __nv_bfloat16 *,
                      __nv_bfloat16 *, long, int, float);

#define BN_ACTS(K, V) {K<V, PCNN_ACT_NONE>, K<V, PCNN_ACT_RELU>, K<V, PCNN_ACT_SILU>, K<V, PCNN_ACT_HARDSWISH>, K<V, PCNN_ACT_RELU6>}

// both backward entries: the reduce pass, the fixed-order slot sums into dbeta and dgamma, the dx pass.  y is read at act 3, beta
// and r at codes 4-6.
int bn_bwd_launch(pcnn_ctx *ctx, const BnGeom &gm, const void *x_bf16, const void *y_bf16, const void *r_bf16, const void *dy_bf16,
                  const void *dy2_bf16, const float *gamma, const float *beta, const float *save_mean, const float *save_rstd, void *dx_bf16,
                  void *dr_bf16, float *dgamma, float *dbeta, long pixels, int C, int act) {
    pcnn_device_guard dg(ctx->device);
    float *slots = nullptr;
    int rc;
    if ((rc = pcnn_scratch(ctx, (size_t)2 * gm.ctas * C * sizeof(float), (void **)&slots))) return rc;
    const auto *x = static_cast<const __nv_bfloat16 *>(x_bf16);
    const auto *y = static_cast<const __nv_bfloat16 *>(y_bf16);
    const auto *r = static_cast<const __nv_bfloat16 *>(r_bf16);
    const auto *dy = static_cast<const __nv_bfloat16 *>(dy_bf16);
    const auto *dy2 = static_cast<const __nv_bfloat16 *>(dy2_bf16);
    const int v8 = gm.vec == 8 ? 1 : 0, col = act_col(act);
    static const reduce_fn rtable[2][5] = {BN_ACTS(k_bn_bwd_reduce, 1), BN_ACTS(k_bn_bwd_reduce, 8)};
    rtable[v8][col]<<<(unsigned)gm.ctas, BN_THREADS, 0, ctx->stream>>>(x, y, r, dy, dy2, save_mean, save_rstd, gamma, beta, slots, pixels, C,
                                                                       gm.ctas);
    PCNN_CHECK_LAUNCH(ctx);
    if ((rc = pcnn_conv_wgrad_reduce_slots(ctx, slots, dbeta, (int)gm.ctas, C))) return rc;
    if ((rc = pcnn_conv_wgrad_reduce_slots(ctx, slots + gm.ctas * C, dgamma, (int)gm.ctas, C))) return rc;
    static const dx_fn dtable[2][5] = {BN_ACTS(k_bn_bwd_dx, 1), BN_ACTS(k_bn_bwd_dx, 8)};
    dtable[v8][col]<<<(unsigned)gm.ctas, BN_THREADS, 0, ctx->stream>>>(x, y, r, dy, dy2, save_mean, save_rstd, gamma, beta, dgamma, dbeta,
                                                                       static_cast<__nv_bfloat16 *>(dx_bf16),
                                                                       static_cast<__nv_bfloat16 *>(dr_bf16), pixels, C, (float)pixels);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

}  // namespace

extern "C" int pcnn_batchnorm_nhwc_info(long pixels, int C, int training, int *out5) {
    const char *fn = "pcnn_batchnorm_nhwc_info";
    PCNN_REQUIRE(out5, PCNN_ERR_ARG, "%s: NULL out5", fn);
    BnGeom gm;
    int rc = bn_geom(fn, pixels, C, training, &gm);
    if (rc) return rc;
    out5[0] = gm.vec;
    out5[1] = gm.lanes;
    out5[2] = (int)gm.per_cta;
    out5[3] = training ? (int)gm.ctas : 0;
    out5[4] = (int)gm.ctas;
    return PCNN_OK;
}

extern "C" int pcnn_batchnorm_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16, const void *r_bf16, void *y_bf16, long pixels, int C, int act,
                                            int training, float eps, float momentum, const float *gamma, const float *beta,
                                            float *running_mean, float *running_var, float *save_mean, float *save_rstd) {
    const char *fn = "pcnn_batchnorm_nhwc_bf16_fwd";
    PCNN_REQUIRE(ctx && x_bf16 && y_bf16 && gamma && beta, PCNN_ERR_ARG, "%s: NULL context, x, y, gamma or beta (only r may be NULL)", fn);
    int rc = bn_act(fn, act, BN_FWD);
    if (rc) return rc;
    BnGeom gm;
    if ((rc = bn_geom(fn, pixels, C, training, &gm))) return rc;
    PCNN_REQUIRE(isfinite(eps) && eps >= 0.0f, PCNN_ERR_ARG, "%s: eps = %g: a finite eps >= 0 is required", fn, (double)eps);
    PCNN_REQUIRE(momentum >= 0.0f && momentum <= 1.0f, PCNN_ERR_ARG, "%s: momentum = %g: 0 <= momentum <= 1 is required", fn,
                 (double)momentum);
    if (training) {
        PCNN_REQUIRE(save_mean && save_rstd, PCNN_ERR_ARG, "%s: training needs save_mean and save_rstd (NULL given)", fn);
        PCNN_REQUIRE(!running_mean == !running_var, PCNN_ERR_ARG, "%s: running_mean and running_var must both be given or both be NULL",
                     fn);
    } else {
        PCNN_REQUIRE(running_mean && running_var, PCNN_ERR_ARG, "%s: eval (training = 0) needs running_mean and running_var (NULL given)", fn);
    }
    const void *ptrs[9] = {x_bf16, r_bf16, y_bf16, gamma, beta, running_mean, running_var, save_mean, save_rstd};
    for (const void *q : ptrs)
        PCNN_REQUIRE(aligned16(q), PCNN_ERR_ARG, "%s: x, r, y, gamma, beta and the statistics must be 16-byte aligned", fn);
    const size_t tb = (size_t)pixels * C * 2, cb = (size_t)C * sizeof(float);
    const Buf bufs[9] = {{x_bf16, tb}, {r_bf16, tb}, {y_bf16, tb}, {gamma, cb}, {beta, cb}, {running_mean, cb}, {running_var, cb},
                         {training ? save_mean : nullptr, cb}, {training ? save_rstd : nullptr, cb}};
    PCNN_REQUIRE(disjoint(bufs, 9), PCNN_ERR_ARG, "%s: overlapping buffers: x, r, y, gamma, beta and the statistics must not share memory", fn);
    pcnn_device_guard dg(ctx->device);
    const auto *x = static_cast<const __nv_bfloat16 *>(x_bf16);
    const auto *r = static_cast<const __nv_bfloat16 *>(r_bf16);
    auto *y = static_cast<__nv_bfloat16 *>(y_bf16);
    const int v8 = gm.vec == 8 ? 1 : 0;
    if (training) {
        float *slots = nullptr;
        if ((rc = pcnn_scratch(ctx, (size_t)3 * gm.ctas * C * sizeof(float), (void **)&slots))) return rc;
        if (v8)
            k_bn_stats<8><<<(unsigned)gm.ctas, BN_THREADS, 0, ctx->stream>>>(x, slots, pixels, C, gm.ctas);
        else
            k_bn_stats<1><<<(unsigned)gm.ctas, BN_THREADS, 0, ctx->stream>>>(x, slots, pixels, C, gm.ctas);
        PCNN_CHECK_LAUNCH(ctx);
        k_bn_finalize<<<(C + 31) / 32, 32 * FIN_ROWS, 0, ctx->stream>>>(slots, gm.ctas, pixels, C, gm.per_cta, eps, momentum, save_mean, save_rstd,
                                                              running_mean, running_var);
        PCNN_CHECK_LAUNCH(ctx);
    }
    static const apply_fn table[2][5] = {BN_ACTS(k_bn_apply, 1), BN_ACTS(k_bn_apply, 8)};
    table[v8][act_col(act)]<<<(unsigned)gm.ctas, BN_THREADS, 0, ctx->stream>>>(x, r, y, training ? save_mean : running_mean,
                                                                       training ? save_rstd : nullptr, training ? nullptr : running_var, eps,
                                                                       gamma, beta, pixels, C);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_batchnorm_nhwc_bf16_bwd(pcnn_ctx *ctx, const void *x_bf16, const void *y_bf16, const void *dy_bf16, const void *dy2_bf16,
                                            const float *gamma, const float *save_mean, const float *save_rstd, void *dx_bf16, void *dr_bf16,
                                            float *dgamma, float *dbeta, long pixels, int C, int act) {
    const char *fn = "pcnn_batchnorm_nhwc_bf16_bwd";
    PCNN_REQUIRE(ctx && x_bf16 && y_bf16 && dy_bf16 && gamma && save_mean && save_rstd && dx_bf16 && dgamma && dbeta, PCNN_ERR_ARG,
                 "%s: NULL context, x, y, dy, gamma, save_mean, save_rstd, dx, dgamma or dbeta (only dy2 and dr may be NULL)", fn);
    int rc = bn_act(fn, act, BN_BWD);
    if (rc) return rc;
    BnGeom gm;
    if ((rc = bn_geom(fn, pixels, C, 1, &gm))) return rc;
    const void *ptrs[11] = {x_bf16, y_bf16, dy_bf16, dy2_bf16, gamma, save_mean, save_rstd, dx_bf16, dr_bf16, dgamma, dbeta};
    for (const void *q : ptrs)
        PCNN_REQUIRE(aligned16(q), PCNN_ERR_ARG, "%s: x, y, dy, dy2, dx, dr, gamma, dgamma, dbeta and the statistics must be 16-byte aligned", fn);
    const size_t tb = (size_t)pixels * C * 2, cb = (size_t)C * sizeof(float);
    const Buf bufs[11] = {{x_bf16, tb},    {y_bf16, tb},    {dy_bf16, tb}, {dy2_bf16, tb}, {gamma, cb}, {save_mean, cb},
                          {save_rstd, cb}, {dx_bf16, tb},   {dr_bf16, tb}, {dgamma, cb},   {dbeta, cb}};
    PCNN_REQUIRE(disjoint(bufs, 11, dx_bf16, dy_bf16), PCNN_ERR_ARG,
                 "%s: overlapping buffers: only dx == dy (in place) may share memory", fn);
    return bn_bwd_launch(ctx, gm, x_bf16, y_bf16, nullptr, dy_bf16, dy2_bf16, gamma, nullptr, save_mean, save_rstd, dx_bf16, dr_bf16, dgamma,
                         dbeta, pixels, C, act);
}

extern "C" int pcnn_batchnorm_nhwc_bf16_bwd_preact(pcnn_ctx *ctx, const void *x_bf16, const void *r_bf16, const void *dy_bf16,
                                                   const void *dy2_bf16, const float *gamma, const float *beta, const float *save_mean,
                                                   const float *save_rstd, void *dx_bf16, void *dr_bf16, float *dgamma, float *dbeta, long pixels,
                                                   int C, int act) {
    const char *fn = "pcnn_batchnorm_nhwc_bf16_bwd_preact";
    PCNN_REQUIRE(ctx && x_bf16 && dy_bf16 && gamma && beta && save_mean && save_rstd && dx_bf16 && dgamma && dbeta, PCNN_ERR_ARG,
                 "%s: NULL context, x, dy, gamma, beta, save_mean, save_rstd, dx, dgamma or dbeta (only r, dy2 and dr may be NULL)", fn);
    int rc = bn_act(fn, act, BN_BWD_PREACT);
    if (rc) return rc;
    BnGeom gm;
    if ((rc = bn_geom(fn, pixels, C, 1, &gm))) return rc;
    const void *ptrs[12] = {x_bf16, r_bf16, dy_bf16, dy2_bf16, gamma, beta, save_mean, save_rstd, dx_bf16, dr_bf16, dgamma, dbeta};
    for (const void *q : ptrs)
        PCNN_REQUIRE(aligned16(q), PCNN_ERR_ARG,
                     "%s: x, r, dy, dy2, dx, dr, gamma, beta, dgamma, dbeta and the statistics must be 16-byte aligned", fn);
    const size_t tb = (size_t)pixels * C * 2, cb = (size_t)C * sizeof(float);
    const Buf bufs[12] = {{x_bf16, tb}, {r_bf16, tb},    {dy_bf16, tb},   {dy2_bf16, tb}, {gamma, cb},  {beta, cb},
                          {save_mean, cb}, {save_rstd, cb}, {dx_bf16, tb}, {dr_bf16, tb},  {dgamma, cb}, {dbeta, cb}};
    PCNN_REQUIRE(disjoint(bufs, 12, dx_bf16, dy_bf16), PCNN_ERR_ARG,
                 "%s: overlapping buffers: only dx == dy (in place) may share memory", fn);
    return bn_bwd_launch(ctx, gm, x_bf16, nullptr, r_bf16, dy_bf16, dy2_bf16, gamma, beta, save_mean, save_rstd, dx_bf16, dr_bf16, dgamma,
                         dbeta, pixels, C, act);
}
