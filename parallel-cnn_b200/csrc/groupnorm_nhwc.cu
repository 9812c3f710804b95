// parallel-cnn_b200/csrc/groupnorm_nhwc.cu -- group normalization of the dense bf16 NHWC [N][H W][C] activations the conv forwards
// write (pcnn_groupnorm_nhwc_bf16_fwd / _bwd / _bwd_preact), with batch normalization's residual add and activations fused into the
// elementwise pass.  The statistics are keyed by (image, group), the parameter gradients by channel; the contract, every
// operation in its order, is in include/pcnn.h.
//
// Partition, a function of (H W, C, G) alone: with C % 8 == 0 a thread moves 16-byte vectors of 8 channels of one pixel, otherwise
// single elements (VEC).  The C / VEC channel groups are cut into slices of at most 256 channels (Gc groups); the H W pixels of an
// image into ranges of GN_ITERS * lanes pixels (lanes = 256 / Gc).  CTA (n, range, slice) owns those pixels and channels; thread t
// keeps channel group t % Gc of the pixels lane, lane + lanes, ... of the range (lane = t / Gc), so consecutive threads touch
// consecutive bytes.  Every pass over the elements runs this grid.
//
// Both reductions go through per-(image, range, channel) fp32 slots in the context's scratch block, so that one set of partials
// serves the per-(image, group) and the per-channel keys and a group may cut across a vector (Cg < 8) or a slice:
//   - forward: k_gn_stats writes {k, sum d, sum d^2} per slot, d = x - k, k the range's first pixel (a shift taken from the data,
//     as batch normalization's); k_gn_finalize gives each (n, g) one warp, which merges the Cg x ranges slots of the group in
//     double in a fixed order (Chan's formula in two passes) into save_mean and save_rstd; k_gn_apply reads x a second time.
//   - backward: k_gn_bwd_reduce writes {sum g, sum g * xhat} per slot; pcnn_conv_wgrad_reduce_slots adds them over (n, range)
//     into dbeta and dgamma, and k_gn_group weighs them with gamma and adds them over (c in g, range) in double into
//     dstat = {A, B}; k_gn_bwd_dx reads dstat back.
// No atomics and nothing depends on the SM count or on N: reruns, every H100 and every batch position give the same bits per image.
#include "pcnn_internal.h"
#include "tc_common.cuh"

#include <cuda_bf16.h>

#include <math.h>

namespace {

constexpr int GN_THREADS = 256;
constexpr int GN_ITERS = 8;          // pixels per thread
constexpr int GN_MIN_CTAS = 2;
constexpr int GN_SLICE_C = 256;      // channels of a slice
constexpr int GN_MAX_C = 2048;
constexpr int GN_WARPS = 8;          // (image, group) pairs per CTA of the merge passes

#include "norm_act.cuh"

// where CTA blockIdx.x works: image n, pixels [p0, p1) of it, channels [c0, c0 + Gc * VEC) (fewer in the last slice)
struct GnCta {
    int n, slice, range, p0, p1, c0, nc;
};

__device__ __forceinline__ GnCta gn_cta(int HW, int C, int VEC, int Gc, int slices, int ranges, int per_cta) {
    GnCta t;
    long b = blockIdx.x;
    t.slice = (int)(b % slices);
    b /= slices;
    t.range = (int)(b % ranges);
    t.n = (int)(b / ranges);
    t.p0 = t.range * per_cta;
    t.p1 = min(HW, t.p0 + per_cta);
    t.c0 = t.slice * Gc * VEC;
    t.nc = min(Gc * VEC, C - t.c0);
    return t;
}

// per-CTA sums of the lanes of two [lanes][nc] planes in lane order -> slot planes [which][(n ranges + range)][C] of `plane` floats
__device__ __forceinline__ void gn_cta_sums(const float *part, int lanes, const GnCta &t, int C, int ranges, float *slots, long plane) {
    const long row = ((long)t.n * ranges + t.range) * C + t.c0;
    for (int i = threadIdx.x; i < 2 * t.nc; i += GN_THREADS) {
        const int which = i / t.nc, c = i - which * t.nc;
        const float *p = part + which * GN_THREADS * 8;
        float s = 0.0f;
        for (int l = 0; l < lanes; ++l) s = __fadd_rn(s, p[l * t.nc + c]);
        slots[which * plane + row + c] = s;
    }
}

struct GnArgs {
    int N, HW, C, G, Cg;
    int Gc, slices, lanes, per_cta, ranges;
    long plane;               // floats of one slot plane: N ranges C
};

template <int VEC>
__global__ void __launch_bounds__(GN_THREADS, GN_MIN_CTAS) k_gn_stats(const __nv_bfloat16 *__restrict__ x, float *__restrict__ slots, GnArgs a) {
    __shared__ float part[2 * GN_THREADS * 8];        // two [lanes][nc] planes: lanes * nc <= 256 * VEC
    constexpr int U = bn_unroll<VEC>();
    const GnCta t = gn_cta(a.HW, a.C, VEC, a.Gc, a.slices, a.ranges, a.per_cta);
    const int lane = threadIdx.x / a.Gc, g = threadIdx.x % a.Gc;
    const __nv_bfloat16 *xi = x + (long)t.n * a.HW * a.C + t.c0 + g * VEC;
    if (lane < a.lanes && g * VEC < t.nc) {
        const BfVec<VEC> kv = ld<VEC>(xi + (long)t.p0 * a.C);     // the range's first pixel: every thread's shift
        float k[VEC], s1[VEC], s2[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
            k[i] = __bfloat162float(kv.h[i]);
            s1[i] = s2[i] = 0.0f;
        }
        for (int j0 = 0; j0 < GN_ITERS; j0 += U) {
            BfVec<VEC> v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int px = t.p0 + lane + (j0 + u) * a.lanes;
                if (px < t.p1) v[u] = ld<VEC>(xi + (long)px * a.C);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (t.p0 + lane + (j0 + u) * a.lanes >= t.p1) continue;
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
            part[lane * t.nc + g * VEC + i] = s1[i];
            part[GN_THREADS * 8 + lane * t.nc + g * VEC + i] = s2[i];
        }
    }
    __syncthreads();
    gn_cta_sums(part, a.lanes, t, a.C, a.ranges, slots + a.plane, a.plane);          // planes 1 and 2: sum d, sum d^2
    const long row = ((long)t.n * a.ranges + t.range) * a.C + t.c0;
    for (int c = threadIdx.x; c < t.nc; c += GN_THREADS)                              // plane 0: k
        slots[row + c] = __bfloat162float(x[((long)t.n * a.HW + t.p0) * a.C + t.c0 + c]);
}

// the sum of the 32 lanes' v in a fixed butterfly: every lane ends with the same bits (a + b == b + a)
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int s = 16; s >= 1; s /= 2) v += __shfl_xor_sync(0xffffffffu, v, s);
    return v;
}

// one warp per (n, g): lane l walks the slots j = l, l + 32, ... of the group, j = (c - g Cg) ranges + range, in double
__global__ void __launch_bounds__(32 * GN_WARPS) k_gn_finalize(const float *__restrict__ slots, GnArgs a, float eps, float *__restrict__ save_mean,
                                                              float *__restrict__ save_rstd) {
    const long ng = (long)blockIdx.x * GN_WARPS + threadIdx.x / 32;
    if (ng >= (long)a.N * a.G) return;
    const int n = (int)(ng / a.G), grp = (int)(ng % a.G), l = threadIdx.x & 31;
    const int terms = a.Cg * a.ranges;
    const float *K = slots, *S1 = slots + a.plane, *S2 = slots + 2 * a.plane;
    auto at = [&](int j, double *nb) {
        const int c = grp * a.Cg + j / a.ranges, b = j % a.ranges;
        *nb = (double)min(a.per_cta, a.HW - b * a.per_cta);
        return ((long)n * a.ranges + b) * a.C + c;
    };
    double s = 0.0, nb;
    for (int j = l; j < terms; j += 32) {
        const long i = at(j, &nb);
        s += nb * (double)K[i] + (double)S1[i];
    }
    const double Mg = (double)a.HW * a.Cg;
    const double mean = warp_sum(s) / Mg;
    s = 0.0;
    for (int j = l; j < terms; j += 32) {
        const long i = at(j, &nb);
        const double s1 = (double)S1[i];
        const double d = ((double)K[i] + s1 / nb) - mean;
        s += ((double)S2[i] - s1 * (s1 / nb)) + nb * d * d;
    }
    const double m2 = fmax(warp_sum(s), 0.0);
    if (l != 0) return;
    save_mean[ng] = (float)mean;
    save_rstd[ng] = (float)__drcp_rn(__dsqrt_rn(m2 / Mg + (double)eps));
}

// the per-channel constants of the CTA's slice in shared memory, local channel c of group (t.c0 + c) / Cg of image n
__device__ __forceinline__ void gn_consts(const GnCta &t, const GnArgs &a, const float *mean, const float *rstd, const float *gamma,
                                          const float *beta, float *mu, float *rs, float *ga, float *be) {
    for (int c = threadIdx.x; c < t.nc; c += GN_THREADS) {
        const long ng = (long)t.n * a.G + (t.c0 + c) / a.Cg;
        mu[c] = mean[ng];
        rs[c] = rstd[ng];
        ga[c] = gamma[t.c0 + c];
        if (beta) be[c] = beta[t.c0 + c];
    }
}

// y = bf16_rn(act(xhat * gamma + beta (+ float(r)))) with the (image, group) statistics
template <int VEC, int ACT>
__global__ void __launch_bounds__(GN_THREADS, GN_MIN_CTAS) k_gn_apply(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ r,
                                                         __nv_bfloat16 *__restrict__ y, const float *__restrict__ mean,
                                                         const float *__restrict__ rstd, const float *__restrict__ gamma,
                                                         const float *__restrict__ beta, GnArgs a) {
    __shared__ float mu[GN_SLICE_C], rs[GN_SLICE_C], ga[GN_SLICE_C], be[GN_SLICE_C];
    constexpr int U = bn_unroll<VEC>();
    const GnCta t = gn_cta(a.HW, a.C, VEC, a.Gc, a.slices, a.ranges, a.per_cta);
    gn_consts(t, a, mean, rstd, gamma, beta, mu, rs, ga, be);
    __syncthreads();
    const int lane = threadIdx.x / a.Gc, g = threadIdx.x % a.Gc;
    if (lane >= a.lanes || g * VEC >= t.nc) return;
    const long base = (long)t.n * a.HW * a.C + t.c0 + g * VEC;
    for (int j0 = 0; j0 < GN_ITERS; j0 += U) {
        BfVec<VEC> xv[U], rv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int px = t.p0 + lane + (j0 + u) * a.lanes;
            if (px < t.p1) {
                xv[u] = ld<VEC>(x + base + (long)px * a.C);
                if (r) rv[u] = ld<VEC>(r + base + (long)px * a.C);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int px = t.p0 + lane + (j0 + u) * a.lanes;
            if (px >= t.p1) continue;
            BfVec<VEC> out;
#pragma unroll
            for (int i = 0; i < VEC; ++i) {
                const int c = g * VEC + i;
                out.h[i] = __float2bfloat16_rn(bn_act_f32<ACT>(bn_pre(bn_xhat(xv[u].h[i], mu[c], rs[c]), ga[c], be[c], r, rv[u].h[i])));
            }
            st<VEC>(y + base + (long)px * a.C, out);
        }
    }
}

// first backward pass: slots [0] = sum g~, [1] = sum g~ * xhat per (image, range, channel).  At codes 4-6 g~ comes from the
// pre-activation recomputed from x, beta and r (y is not read).
template <int VEC, int ACT>
__global__ void __launch_bounds__(GN_THREADS, GN_MIN_CTAS) k_gn_bwd_reduce(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ y,
                                                              const __nv_bfloat16 *__restrict__ r, const __nv_bfloat16 *__restrict__ dy,
                                                              const __nv_bfloat16 *__restrict__ dy2, const float *__restrict__ mean,
                                                              const float *__restrict__ rstd, const float *__restrict__ gamma,
                                                              const float *__restrict__ beta, float *__restrict__ slots, GnArgs a) {
    constexpr bool PRE = bn_preact<ACT>();
    __shared__ float part[2 * GN_THREADS * 8];
    __shared__ float mu[GN_SLICE_C], rs[GN_SLICE_C], ga[PRE ? GN_SLICE_C : 1], be[PRE ? GN_SLICE_C : 1];
    constexpr int U = bn_unroll<VEC>();
    const GnCta t = gn_cta(a.HW, a.C, VEC, a.Gc, a.slices, a.ranges, a.per_cta);
    for (int c = threadIdx.x; c < t.nc; c += GN_THREADS) {
        const long ng = (long)t.n * a.G + (t.c0 + c) / a.Cg;
        mu[c] = mean[ng];
        rs[c] = rstd[ng];
        if (PRE) {
            ga[c] = gamma[t.c0 + c];
            be[c] = beta[t.c0 + c];
        }
    }
    __syncthreads();
    const int lane = threadIdx.x / a.Gc, g = threadIdx.x % a.Gc;
    if (lane < a.lanes && g * VEC < t.nc) {
        const long base = (long)t.n * a.HW * a.C + t.c0 + g * VEC;
        float sb[VEC], sg[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) sb[i] = sg[i] = 0.0f;
        for (int j0 = 0; j0 < GN_ITERS; j0 += U) {
            BfVec<VEC> xv[U], yv[U], dv[U], d2[U], rv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int px = t.p0 + lane + (j0 + u) * a.lanes;
                if (px < t.p1) {
                    const long off = base + (long)px * a.C;
                    xv[u] = ld<VEC>(x + off);
                    dv[u] = ld<VEC>(dy + off);
                    if (ACT == PCNN_ACT_RELU) yv[u] = ld<VEC>(y + off);
                    if (PRE && r) rv[u] = ld<VEC>(r + off);
                    if (dy2) d2[u] = ld<VEC>(dy2 + off);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (t.p0 + lane + (j0 + u) * a.lanes >= t.p1) continue;
#pragma unroll
                for (int i = 0; i < VEC; ++i) {
                    const int c = g * VEC + i;
                    const float xh = bn_xhat(xv[u].h[i], mu[c], rs[c]);
                    float gt;
                    if constexpr (PRE)
                        gt = __bfloat162float(bn_dgrad_pre<ACT>(dv[u].h[i], d2[u].h[i], dy2 != nullptr, bn_pre(xh, ga[c], be[c], r, rv[u].h[i])));
                    else
                        gt = __bfloat162float(bn_dgrad<ACT>(dv[u].h[i], d2[u].h[i], dy2 != nullptr, yv[u].h[i]));
                    sb[i] = __fadd_rn(sb[i], gt);
                    sg[i] = __fadd_rn(sg[i], __fmul_rn(gt, xh));
                }
            }
        }
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
            part[lane * t.nc + g * VEC + i] = sb[i];
            part[GN_THREADS * 8 + lane * t.nc + g * VEC + i] = sg[i];
        }
    }
    __syncthreads();
    gn_cta_sums(part, a.lanes, t, a.C, a.ranges, slots, a.plane);
}

// one warp per (n, g): A = sum gamma[c] * slot0, B = sum gamma[c] * slot1 over the group's slots in double (each product is exact),
// lane l taking j = l, l + 32, ... as k_gn_finalize; dstat[0][n][g] = float(A), dstat[1][n][g] = float(B)
__global__ void __launch_bounds__(32 * GN_WARPS) k_gn_group(const float *__restrict__ slots, const float *__restrict__ gamma, GnArgs a,
                                                           float *__restrict__ dstat) {
    const long ng = (long)blockIdx.x * GN_WARPS + threadIdx.x / 32;
    if (ng >= (long)a.N * a.G) return;
    const int n = (int)(ng / a.G), grp = (int)(ng % a.G), l = threadIdx.x & 31;
    double sa = 0.0, sb = 0.0;
    for (int j = l; j < a.Cg * a.ranges; j += 32) {
        const int c = grp * a.Cg + j / a.ranges, b = j % a.ranges;
        const long i = ((long)n * a.ranges + b) * a.C + c;
        const double w = (double)gamma[c];
        sa += w * (double)slots[i];
        sb += w * (double)slots[a.plane + i];
    }
    sa = warp_sum(sa);
    sb = warp_sum(sb);
    if (l != 0) return;
    dstat[ng] = (float)sa;
    dstat[(long)a.N * a.G + ng] = (float)sb;
}

// second backward pass: dx = bf16_rn(((g~ * gamma - A / Mgf) - xhat * (B / Mgf)) * rstd), dr = g~.  dx may be dy.
template <int VEC, int ACT>
__global__ void __launch_bounds__(GN_THREADS, GN_MIN_CTAS) k_gn_bwd_dx(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ y,
                                                          const __nv_bfloat16 *__restrict__ r, const __nv_bfloat16 *dy,
                                                          const __nv_bfloat16 *__restrict__ dy2, const float *__restrict__ mean,
                                                          const float *__restrict__ rstd, const float *__restrict__ gamma,
                                                          const float *__restrict__ beta, const float *__restrict__ dstat, __nv_bfloat16 *dx,
                                                          __nv_bfloat16 *__restrict__ dr, GnArgs a, float Mgf) {
    constexpr bool PRE = bn_preact<ACT>();
    constexpr int U = bn_unroll<VEC>();
    __shared__ float mu[GN_SLICE_C], rs[GN_SLICE_C], ga[GN_SLICE_C], be[PRE ? GN_SLICE_C : 1], ma[GN_SLICE_C], mb[GN_SLICE_C];
    const GnCta t = gn_cta(a.HW, a.C, VEC, a.Gc, a.slices, a.ranges, a.per_cta);
    const long NG = (long)a.N * a.G;
    for (int c = threadIdx.x; c < t.nc; c += GN_THREADS) {
        const long ng = (long)t.n * a.G + (t.c0 + c) / a.Cg;
        mu[c] = mean[ng];
        rs[c] = rstd[ng];
        ga[c] = gamma[t.c0 + c];
        if (PRE) be[c] = beta[t.c0 + c];
        ma[c] = __fdiv_rn(dstat[ng], Mgf);
        mb[c] = __fdiv_rn(dstat[NG + ng], Mgf);
    }
    __syncthreads();
    const int lane = threadIdx.x / a.Gc, g = threadIdx.x % a.Gc;
    if (lane >= a.lanes || g * VEC >= t.nc) return;
    const long base = (long)t.n * a.HW * a.C + t.c0 + g * VEC;
    for (int j0 = 0; j0 < GN_ITERS; j0 += U) {
        BfVec<VEC> xv[U], yv[U], dv[U], d2[U], rv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int px = t.p0 + lane + (j0 + u) * a.lanes;
            if (px < t.p1) {
                const long off = base + (long)px * a.C;
                xv[u] = ld<VEC>(x + off);
                dv[u] = ld<VEC>(dy + off);
                if (ACT == PCNN_ACT_RELU) yv[u] = ld<VEC>(y + off);
                if (PRE && r) rv[u] = ld<VEC>(r + off);
                if (dy2) d2[u] = ld<VEC>(dy2 + off);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int px = t.p0 + lane + (j0 + u) * a.lanes;
            if (px >= t.p1) continue;
            BfVec<VEC> o, gv;
#pragma unroll
            for (int i = 0; i < VEC; ++i) {
                const int c = g * VEC + i;
                const float xh = bn_xhat(xv[u].h[i], mu[c], rs[c]);
                if constexpr (PRE)
                    gv.h[i] = bn_dgrad_pre<ACT>(dv[u].h[i], d2[u].h[i], dy2 != nullptr, bn_pre(xh, ga[c], be[c], r, rv[u].h[i]));
                else
                    gv.h[i] = bn_dgrad<ACT>(dv[u].h[i], d2[u].h[i], dy2 != nullptr, yv[u].h[i]);
                const float v = __fsub_rn(__fsub_rn(__fmul_rn(__bfloat162float(gv.h[i]), ga[c]), ma[c]), __fmul_rn(xh, mb[c]));
                o.h[i] = __float2bfloat16_rn(__fmul_rn(v, rs[c]));
            }
            const long off = base + (long)px * a.C;
            st<VEC>(dx + off, o);
            if (dr) st<VEC>(dr + off, gv);
        }
    }
}

struct GnGeom {
    int vec;
    long ctas, group_ctas;
    GnArgs a;
};

// the shape rules of pcnn.h, refused with PCNN_ERR_ARG and a message naming `fn`; the partition depends on (HW, C, G) alone
int gn_geom(const char *fn, int N, int HW, int C, int G, GnGeom *out) {
    PCNN_REQUIRE(N >= 1, PCNN_ERR_ARG, "%s: N = %d images: N >= 1 is required", fn, N);
    PCNN_REQUIRE(HW >= 1, PCNN_ERR_ARG, "%s: HW = %d pixels per image: H * W >= 1 is required", fn, HW);
    PCNN_REQUIRE(C >= 1 && C <= GN_MAX_C, PCNN_ERR_ARG, "%s: C = %d channels: 1 <= C <= 2048 is required", fn, C);
    PCNN_REQUIRE(G >= 1 && G <= C && C % G == 0, PCNN_ERR_ARG, "%s: G = %d groups of C = %d channels: 1 <= G <= C with C %% G == 0 is required",
                 fn, G, C);
    GnArgs &a = out->a;
    out->vec = C % 8 == 0 ? 8 : 1;
    a.N = N;
    a.HW = HW;
    a.C = C;
    a.G = G;
    a.Cg = C / G;
    const int groups = C / out->vec;
    a.Gc = groups < GN_SLICE_C / out->vec ? groups : GN_SLICE_C / out->vec;
    a.slices = (groups + a.Gc - 1) / a.Gc;
    a.lanes = GN_THREADS / a.Gc;
    a.per_cta = GN_ITERS * a.lanes;
    a.ranges = (HW + a.per_cta - 1) / a.per_cta;
    out->ctas = (long)N * a.ranges * a.slices;
    a.plane = (long)N * a.ranges * C;
    out->group_ctas = ((long)N * G + GN_WARPS - 1) / GN_WARPS;
    PCNN_REQUIRE(out->ctas < (1L << 31) && (long)N * a.ranges < (1L << 31), PCNN_ERR_ARG,
                 "%s: N = %d images of HW = %d pixels exceed the grid (N * ranges * slices < 2^31 CTAs is required)", fn, N, HW);
    return PCNN_OK;
}

enum GnPass { GN_FWD, GN_BWD, GN_BWD_PREACT };

bool act_from_preact(int act) { return act == PCNN_ACT_SILU || act == PCNN_ACT_HARDSWISH || act == PCNN_ACT_RELU6; }

// the codes each entry takes: the forward 0 and 3-6, the backward 0 and 3, the pre-activation backward 4-6
int gn_act(const char *fn, int act, GnPass pass) {
    PCNN_REQUIRE(act != PCNN_ACT_SIGMOID, PCNN_ERR_ARG,
                 "%s: act 1 (sigmoid) is not available after group normalization: sigmoid_bf16 uses tanh.approx, which no reference "
                 "can replay bit for bit; %s is required", fn,
                 pass == GN_BWD_PREACT ? "act 4 (SiLU), 5 (hard-swish) or 6 (ReLU6)" : "act 0 (none) or 3 (ReLU)");
    const bool plain = act == PCNN_ACT_NONE || act == PCNN_ACT_RELU, pre = act_from_preact(act);
    if (pass == GN_FWD)
        PCNN_REQUIRE(plain || pre, PCNN_ERR_ARG, "%s: act %d is not 0 (none) or 3 (ReLU), nor 4 (SiLU), 5 (hard-swish) or 6 (ReLU6)", fn, act);
    if (pass == GN_BWD) {
        PCNN_REQUIRE(!pre, PCNN_ERR_ARG,
                     "%s: act %d takes its gradient from the recomputed pre-activation, not from y: pcnn_groupnorm_nhwc_bf16_bwd_preact "
                     "is its backward", fn, act);
        PCNN_REQUIRE(plain, PCNN_ERR_ARG, "%s: act %d is not 0 (none) or 3 (ReLU)", fn, act);
    }
    if (pass == GN_BWD_PREACT) {
        PCNN_REQUIRE(!plain, PCNN_ERR_ARG, "%s: act %d takes its gradient from y: pcnn_groupnorm_nhwc_bf16_bwd is its backward", fn, act);
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

// true when no two of the non-NULL buffers share a byte, except dx and dy when they are the same buffer (in place)
bool disjoint(const Buf *b, int n, const void *dx = nullptr, const void *dy = nullptr) {
    for (int i = 0; i < n; ++i)
        for (int j = i + 1; j < n; ++j) {
            if (!b[i].p || !b[j].p) continue;
            const uintptr_t pi = (uintptr_t)b[i].p, pj = (uintptr_t)b[j].p;
            if (!(pi < pj + b[j].n && pj < pi + b[i].n)) continue;
            const bool in_place = dx && b[i].p == b[j].p && b[i].n == b[j].n &&
                                  ((b[i].p == dx && b[j].p == dy) || (b[i].p == dy && b[j].p == dx));
            if (!in_place) return false;
        }
    return true;
}

typedef void (*apply_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, __nv_bfloat16 *, const float *, const float *, const float *,
                         const float *, GnArgs);
typedef void (*reduce_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *,
                          const float *, const float *, const float *, const float *, float *, GnArgs);
typedef void (*dx_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *,
                      const float *, const float *, const float *, const float *, const float *, __nv_bfloat16 *, __nv_bfloat16 *, GnArgs,
                      float);

#define GN_ACTS(K, V) {K<V, PCNN_ACT_NONE>, K<V, PCNN_ACT_RELU>, K<V, PCNN_ACT_SILU>, K<V, PCNN_ACT_HARDSWISH>, K<V, PCNN_ACT_RELU6>}

// both backward entries: the reduce pass, dbeta and dgamma over (n, range), A and B over (c in g, range), the dx pass.  y is read
// at act 3, beta and r at codes 4-6.
int gn_bwd_launch(pcnn_ctx *ctx, const GnGeom &gm, const void *x_bf16, const void *y_bf16, const void *r_bf16, const void *dy_bf16,
                  const void *dy2_bf16, const float *gamma, const float *beta, const float *save_mean, const float *save_rstd, void *dx_bf16,
                  void *dr_bf16, float *dgamma, float *dbeta, float *dstat, int act) {
    pcnn_device_guard dg(ctx->device);
    const GnArgs &a = gm.a;
    float *slots = nullptr;
    int rc;
    if ((rc = pcnn_scratch(ctx, (size_t)2 * a.plane * sizeof(float), (void **)&slots))) return rc;
    const auto *x = static_cast<const __nv_bfloat16 *>(x_bf16);
    const auto *y = static_cast<const __nv_bfloat16 *>(y_bf16);
    const auto *r = static_cast<const __nv_bfloat16 *>(r_bf16);
    const auto *dy = static_cast<const __nv_bfloat16 *>(dy_bf16);
    const auto *dy2 = static_cast<const __nv_bfloat16 *>(dy2_bf16);
    const int v8 = gm.vec == 8 ? 1 : 0, col = act_col(act);
    static const reduce_fn rtable[2][5] = {GN_ACTS(k_gn_bwd_reduce, 1), GN_ACTS(k_gn_bwd_reduce, 8)};
    rtable[v8][col]<<<(unsigned)gm.ctas, GN_THREADS, 0, ctx->stream>>>(x, y, r, dy, dy2, save_mean, save_rstd, gamma, beta, slots, a);
    PCNN_CHECK_LAUNCH(ctx);
    const int nslots = a.N * a.ranges;
    if ((rc = pcnn_conv_wgrad_reduce_slots(ctx, slots, dbeta, nslots, a.C))) return rc;
    if ((rc = pcnn_conv_wgrad_reduce_slots(ctx, slots + a.plane, dgamma, nslots, a.C))) return rc;
    k_gn_group<<<(unsigned)gm.group_ctas, 32 * GN_WARPS, 0, ctx->stream>>>(slots, gamma, a, dstat);
    PCNN_CHECK_LAUNCH(ctx);
    static const dx_fn dtable[2][5] = {GN_ACTS(k_gn_bwd_dx, 1), GN_ACTS(k_gn_bwd_dx, 8)};
    dtable[v8][col]<<<(unsigned)gm.ctas, GN_THREADS, 0, ctx->stream>>>(x, y, r, dy, dy2, save_mean, save_rstd, gamma, beta, dstat,
                                                                       static_cast<__nv_bfloat16 *>(dx_bf16),
                                                                       static_cast<__nv_bfloat16 *>(dr_bf16), a, (float)((double)a.HW * a.Cg));
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

}  // namespace

extern "C" int pcnn_groupnorm_nhwc_info(int N, int HW, int C, int G, int *out11) {
    const char *fn = "pcnn_groupnorm_nhwc_info";
    PCNN_REQUIRE(out11, PCNN_ERR_ARG, "%s: NULL out11", fn);
    GnGeom gm;
    int rc = gn_geom(fn, N, HW, C, G, &gm);
    if (rc) return rc;
    const GnArgs &a = gm.a;
    const long slots = (long)N * a.ranges;
    out11[0] = gm.vec;
    out11[1] = a.Gc;
    out11[2] = a.slices;
    out11[3] = a.lanes;
    out11[4] = a.per_cta;
    out11[5] = a.ranges;
    out11[6] = (int)gm.ctas;
    out11[7] = (int)slots;
    out11[8] = (int)gm.group_ctas;
    out11[9] = GN_ITERS + a.lanes + (int)((slots + 7) / 8) + 3;
    out11[10] = GN_ITERS + a.lanes + 2;
    return PCNN_OK;
}

extern "C" int pcnn_groupnorm_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16, const void *r_bf16, void *y_bf16, int N, int HW, int C, int G,
                                            int act, float eps, const float *gamma, const float *beta, float *save_mean, float *save_rstd) {
    const char *fn = "pcnn_groupnorm_nhwc_bf16_fwd";
    PCNN_REQUIRE(ctx && x_bf16 && y_bf16 && gamma && beta && save_mean && save_rstd, PCNN_ERR_ARG,
                 "%s: NULL context, x, y, gamma, beta, save_mean or save_rstd (only r may be NULL)", fn);
    int rc = gn_act(fn, act, GN_FWD);
    if (rc) return rc;
    GnGeom gm;
    if ((rc = gn_geom(fn, N, HW, C, G, &gm))) return rc;
    PCNN_REQUIRE(isfinite(eps) && eps >= 0.0f, PCNN_ERR_ARG, "%s: eps = %g: a finite eps >= 0 is required", fn, (double)eps);
    const void *ptrs[7] = {x_bf16, r_bf16, y_bf16, gamma, beta, save_mean, save_rstd};
    for (const void *q : ptrs)
        PCNN_REQUIRE(aligned16(q), PCNN_ERR_ARG, "%s: x, r, y, gamma, beta, save_mean and save_rstd must be 16-byte aligned", fn);
    const size_t tb = (size_t)N * HW * C * 2, cb = (size_t)C * sizeof(float), sb = (size_t)N * G * sizeof(float);
    const Buf bufs[7] = {{x_bf16, tb}, {r_bf16, tb}, {y_bf16, tb}, {gamma, cb}, {beta, cb}, {save_mean, sb}, {save_rstd, sb}};
    PCNN_REQUIRE(disjoint(bufs, 7), PCNN_ERR_ARG, "%s: overlapping buffers: x, r, y, gamma, beta and the statistics must not share memory", fn);
    pcnn_device_guard dg(ctx->device);
    const GnArgs &a = gm.a;
    float *slots = nullptr;
    if ((rc = pcnn_scratch(ctx, (size_t)3 * a.plane * sizeof(float), (void **)&slots))) return rc;
    const auto *x = static_cast<const __nv_bfloat16 *>(x_bf16);
    const int v8 = gm.vec == 8 ? 1 : 0;
    if (v8)
        k_gn_stats<8><<<(unsigned)gm.ctas, GN_THREADS, 0, ctx->stream>>>(x, slots, a);
    else
        k_gn_stats<1><<<(unsigned)gm.ctas, GN_THREADS, 0, ctx->stream>>>(x, slots, a);
    PCNN_CHECK_LAUNCH(ctx);
    k_gn_finalize<<<(unsigned)gm.group_ctas, 32 * GN_WARPS, 0, ctx->stream>>>(slots, a, eps, save_mean, save_rstd);
    PCNN_CHECK_LAUNCH(ctx);
    static const apply_fn table[2][5] = {GN_ACTS(k_gn_apply, 1), GN_ACTS(k_gn_apply, 8)};
    table[v8][act_col(act)]<<<(unsigned)gm.ctas, GN_THREADS, 0, ctx->stream>>>(x, static_cast<const __nv_bfloat16 *>(r_bf16),
                                                                               static_cast<__nv_bfloat16 *>(y_bf16), save_mean, save_rstd,
                                                                               gamma, beta, a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_groupnorm_nhwc_bf16_bwd(pcnn_ctx *ctx, const void *x_bf16, const void *y_bf16, const void *dy_bf16, const void *dy2_bf16,
                                            const float *gamma, const float *save_mean, const float *save_rstd, void *dx_bf16, void *dr_bf16,
                                            float *dgamma, float *dbeta, float *dstat, int N, int HW, int C, int G, int act) {
    const char *fn = "pcnn_groupnorm_nhwc_bf16_bwd";
    PCNN_REQUIRE(ctx && x_bf16 && y_bf16 && dy_bf16 && gamma && save_mean && save_rstd && dx_bf16 && dgamma && dbeta && dstat, PCNN_ERR_ARG,
                 "%s: NULL context, x, y, dy, gamma, save_mean, save_rstd, dx, dgamma, dbeta or dstat (only dy2 and dr may be NULL)", fn);
    int rc = gn_act(fn, act, GN_BWD);
    if (rc) return rc;
    GnGeom gm;
    if ((rc = gn_geom(fn, N, HW, C, G, &gm))) return rc;
    const void *ptrs[12] = {x_bf16, y_bf16, dy_bf16, dy2_bf16, gamma, save_mean, save_rstd, dx_bf16, dr_bf16, dgamma, dbeta, dstat};
    for (const void *q : ptrs)
        PCNN_REQUIRE(aligned16(q), PCNN_ERR_ARG,
                     "%s: x, y, dy, dy2, dx, dr, gamma, dgamma, dbeta, dstat and the statistics must be 16-byte aligned", fn);
    const size_t tb = (size_t)N * HW * C * 2, cb = (size_t)C * sizeof(float), sb = (size_t)N * G * sizeof(float);
    const Buf bufs[12] = {{x_bf16, tb},    {y_bf16, tb},  {dy_bf16, tb}, {dy2_bf16, tb}, {gamma, cb}, {save_mean, sb},
                          {save_rstd, sb}, {dx_bf16, tb}, {dr_bf16, tb}, {dgamma, cb},   {dbeta, cb}, {dstat, 2 * sb}};
    PCNN_REQUIRE(disjoint(bufs, 12, dx_bf16, dy_bf16), PCNN_ERR_ARG, "%s: overlapping buffers: only dx == dy (in place) may share memory", fn);
    return gn_bwd_launch(ctx, gm, x_bf16, y_bf16, nullptr, dy_bf16, dy2_bf16, gamma, nullptr, save_mean, save_rstd, dx_bf16, dr_bf16, dgamma,
                         dbeta, dstat, act);
}

extern "C" int pcnn_groupnorm_nhwc_bf16_bwd_preact(pcnn_ctx *ctx, const void *x_bf16, const void *r_bf16, const void *dy_bf16,
                                                   const void *dy2_bf16, const float *gamma, const float *beta, const float *save_mean,
                                                   const float *save_rstd, void *dx_bf16, void *dr_bf16, float *dgamma, float *dbeta,
                                                   float *dstat, int N, int HW, int C, int G, int act) {
    const char *fn = "pcnn_groupnorm_nhwc_bf16_bwd_preact";
    PCNN_REQUIRE(ctx && x_bf16 && dy_bf16 && gamma && beta && save_mean && save_rstd && dx_bf16 && dgamma && dbeta && dstat, PCNN_ERR_ARG,
                 "%s: NULL context, x, dy, gamma, beta, save_mean, save_rstd, dx, dgamma, dbeta or dstat (only r, dy2 and dr may be NULL)",
                 fn);
    int rc = gn_act(fn, act, GN_BWD_PREACT);
    if (rc) return rc;
    GnGeom gm;
    if ((rc = gn_geom(fn, N, HW, C, G, &gm))) return rc;
    const void *ptrs[13] = {x_bf16, r_bf16, dy_bf16, dy2_bf16, gamma, beta, save_mean, save_rstd, dx_bf16, dr_bf16, dgamma, dbeta, dstat};
    for (const void *q : ptrs)
        PCNN_REQUIRE(aligned16(q), PCNN_ERR_ARG,
                     "%s: x, r, dy, dy2, dx, dr, gamma, beta, dgamma, dbeta, dstat and the statistics must be 16-byte aligned", fn);
    const size_t tb = (size_t)N * HW * C * 2, cb = (size_t)C * sizeof(float), sb = (size_t)N * G * sizeof(float);
    const Buf bufs[13] = {{x_bf16, tb},    {r_bf16, tb},    {dy_bf16, tb}, {dy2_bf16, tb}, {gamma, cb},  {beta, cb},    {save_mean, sb},
                          {save_rstd, sb}, {dx_bf16, tb}, {dr_bf16, tb}, {dgamma, cb},   {dbeta, cb}, {dstat, 2 * sb}};
    PCNN_REQUIRE(disjoint(bufs, 13, dx_bf16, dy_bf16), PCNN_ERR_ARG, "%s: overlapping buffers: only dx == dy (in place) may share memory", fn);
    return gn_bwd_launch(ctx, gm, x_bf16, nullptr, r_bf16, dy_bf16, dy2_bf16, gamma, beta, save_mean, save_rstd, dx_bf16, dr_bf16, dgamma,
                         dbeta, dstat, act);
}
