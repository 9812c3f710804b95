// parallel-cnn_b200/csrc/linear_tc.cu -- fully connected layers on the Hopper tensor cores (pcnn_linear_plan_create, run by
// pcnn_conv_tc_fwd; pcnn_linear_wgrad, pcnn_linear_dgrad, pcnn_linear_info) and the bf16 softmax cross-entropy
// (pcnn_softmax_ce_bf16).  sm_90a.
//
// Notation: x is [N][image_rows][row_pitch] bf16 with P x Q pixels of C channels per image (the layout the conv plans and the
// NHWC pool use for an activation); F = P*Q*C features in NHWC order; W the fp32 masters [O][P][Q][C] (KRSC with K = O, R = P,
// S = Q); y and dy dense bf16 [N][O].  The plan keeps W rounded to bf16 as [O][P][wpitch], wpitch = Q*C rounded up to 8.
// A reduction step covers one row p and 64 features of it ("chunk"): P * ceil(Q*C / 64) chunks.
//
//   * Forward  y[n][o] = act(b[o] + sum_f x[n][f] W[o][f]):  M = 128 images per tile (two consumer warpgroups of 64), N = O
//     rounded up to 16, reduction over the chunks.  A: a box {64 features, 1 row, 128 images} of x viewed as {Q*C, P, N}; the
//     inner extent is Q*C, not the pitch, so pad columns and pad rows are never read.  B: a box {64, 1, Npad} of the bf16
//     weights viewed as {Q*C, P, O}, K-major.  Both SWIZZLE_128B.  Split: the chunks are cut into `splits` ranges, each unit
//     (image tile, range) writes fp32 partials into slot [range][N][O] and k_linear_fwd_reduce adds them in range order, then
//     applies bias and activation (none, sigmoid or ReLU: a run-time branch, no extra instantiation).  Unsplit, the epilogue
//     does that from the registers.  y is written with masked stores.
//   * Weight gradient  dW[o][f] = sum_n dy[n][o] x[n][f]:  M = 64 features of one chunk per warpgroup, N = O rounded up to 64,
//     reduction over images, 16 per m64nNk16.  A: the forward's x box (128 image rows of 64 features, MN-major).  B: boxes
//     {64 outputs, 128 images} of dy, MN-major.  A unit is a pair of chunks and a range of 128-image blocks; ranges > 1 write
//     slots [range][O][F] that pcnn_conv_wgrad_reduce_slots adds in order.
//   * Input gradient  dx[n][f] = sum_o dy[n][o] W[o][f]:  M = 128 images, N = up to 4 chunks (256 features), reduction over O
//     in steps of 64.  A: a box {64 outputs, 128 images} of dy, K-major.  B: per chunk a box {64 features, 1 row, 64 outputs}
//     of the plan's bf16 weights, MN-major.  dx is written with masked stores into x's layout; its pad is never written.
//   dy is dense [N][O]; a TMA map needs 16-byte row strides, so for O % 8 != 0 it is first copied into [N][O rounded up to 8]
//   (scratch).  TMA zero-fills outputs >= O, images >= N and features >= Q*C in every box.
// Every split is a function of the shape alone: the bits are the same on every run and every H100.
// Warp roles (288 threads, 1 CTA/SM, persistent over units): warps 0-7 = two consumer warpgroups, warp 8 = TMA producer.
#include "tc_common.cuh"

#include <cuda_bf16.h>
#include <math.h>
#include <memory>

using namespace pcnn_tc;

namespace {

constexpr int LN_THREADS = 288;
constexpr int LN_CONSUMER_WARPS = 8;
constexpr int LN_KC = 64;                        // features / outputs per 128-byte SWIZZLE_128B row
constexpr int LN_M = 128;                        // images per tile
constexpr int LN_BOX = LN_M * LN_KC * 2;         // 128 rows x 64 elements: 16 KB
constexpr int LN_WBOX = 64 * LN_KC * 2;          // 64 outputs x 64 features of the weights: 8 KB
constexpr int LN_MAX_STAGES = 8;
constexpr int LN_SMEM_BUDGET = 225 * 1024;
constexpr int LN_TARGET_UNITS = 128;             // units a split aims for (a constant: never the SM count)
constexpr int LN_MIN_SPLIT_STEPS = 8;            // chunks per forward range, at least
constexpr int LN_DGRAD_MAX_BOXES = 4;            // chunks per input-gradient tile (256 features, the widest wgmma)
constexpr long long LN_MAX_F = 1LL << 24;

struct LnCtl {
    unsigned long long full[LN_MAX_STAGES], empty[LN_MAX_STAGES];
};

__device__ __forceinline__ unsigned char *align1024(unsigned char *p) {
    return reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(p) + 1023) & ~(uintptr_t)1023);
}

__host__ __device__ __forceinline__ int range_begin(int total, int ranges, int r) { return (int)((long long)r * total / ranges); }

// ================================================= forward =====================================================================
struct LinearFwdParams {
    int N, O, nch, steps, splits, mtiles, units, stages, act;
    const float *bias;               // [O] or null
    __nv_bfloat16 *y;                // [N][O] (unsplit)
    float *slots;                    // [splits][N][O] (split)
};

struct LinearMaps {
    CUtensorMap a, b;
};

template <int N>   // accumulator columns: O rounded up to 16
__global__ void __launch_bounds__(LN_THREADS, 1)
k_linear_fwd(const __grid_constant__ LinearMaps m, const LinearFwdParams p) {
    constexpr int B_BYTES = N * LN_KC * 2;
    constexpr int STAGE = LN_BOX + B_BYTES;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *ring = align1024(smem_dyn);
    const int NST = p.stages;
    LnCtl &S = *reinterpret_cast<LnCtl *>(ring + (size_t)NST * STAGE);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int i = 0; i < NST; ++i) { bar_init(&S.full[i], 1); bar_init(&S.empty[i], LN_CONSUMER_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == LN_CONSUMER_WARPS) {
        if (lane == 0) {
            int it = 0;
            for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
                // range-major: the units running together share a range of weights, which L2 serves to every image tile
                const int sp = u / p.mtiles, mt = u % p.mtiles;
                for (int s = range_begin(p.steps, p.splits, sp), s1 = range_begin(p.steps, p.splits, sp + 1); s < s1; ++s, ++it) {
                    const int stage = it % NST;
                    bar_wait_relaxed(&S.empty[stage], ((unsigned)(it / NST) & 1u) ^ 1u, 32);
                    unsigned char *a = ring + (size_t)stage * STAGE;
                    bar_expect_tx(&S.full[stage], (unsigned)STAGE);
                    tma_load_3d(a, &m.a, (s % p.nch) * LN_KC, s / p.nch, mt * LN_M, &S.full[stage]);
                    tma_load_3d(a + LN_BOX, &m.b, (s % p.nch) * LN_KC, s / p.nch, 0, &S.full[stage]);
                }
            }
        }
        return;
    }

    const int wg = warp >> 2, wq = warp & 3;
    int it = 0;
    for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
        const int sp = u / p.mtiles, mt = u % p.mtiles;
        const int nsteps = range_begin(p.steps, p.splits, sp + 1) - range_begin(p.steps, p.splits, sp);
        float acc[N / 2];
        for (int step = 0; step < nsteps; ++step, ++it) {
            const int stage = it % NST;
            bar_wait(&S.full[stage], (unsigned)(it / NST) & 1u);
            const uint32_t a0 = s_u32(ring + (size_t)stage * STAGE) + (uint32_t)(wg * 64 * LN_KC * 2);
            const uint32_t b0 = s_u32(ring + (size_t)stage * STAGE + LN_BOX);
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < LN_KC / 16; ++ks)
                wgmma_bf16<0, 0>(acc, gmma_desc_k_sw128(a0 + ks * 32), gmma_desc_k_sw128(b0 + ks * 32), (step | ks) != 0 ? 1u : 0u);
            wg_commit();
            if (step > 0) {
                wg_wait<1>();
                __syncwarp();
                if (lane == 0) bar_arrive(&S.empty[(it - 1) % NST]);
            }
        }
        wg_wait<0>();
        wg_hold(acc);
        __syncwarp();
        if (lane == 0) bar_arrive(&S.empty[(it - 1) % NST]);
#pragma unroll
        for (int i = 0; i < N / 2; ++i) {
            const int n = mt * LN_M + wg * 64 + wg_row(i, wq, lane), o = wg_col(i, lane);
            if (n >= p.N || o >= p.O) continue;
            if (p.splits > 1) {
                p.slots[((size_t)sp * p.N + n) * p.O + o] = acc[i];
            } else {
                float v = p.bias ? __fadd_rn(acc[i], p.bias[o]) : acc[i];
                if (p.act == PCNN_ACT_SIGMOID) v = sigmoid_bf16(v);
                else if (p.act == PCNN_ACT_RELU) v = relu_f32(v);
                p.y[(size_t)n * p.O + o] = __float2bfloat16_rn(v);
            }
        }
    }
}

// y = act(bias + slots[0] + slots[1] + ...), the slots added in range order
__global__ void __launch_bounds__(256) k_linear_fwd_reduce(const float *__restrict__ slots, int splits, const float *__restrict__ bias,
                                                           int act, __nv_bfloat16 *__restrict__ y, long total, int O) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        float v = slots[i];
        for (int s = 1; s < splits; ++s) v = __fadd_rn(v, slots[(size_t)s * total + i]);
        if (bias) v = __fadd_rn(v, bias[i % O]);
        if (act == PCNN_ACT_SIGMOID) v = sigmoid_bf16(v);
        else if (act == PCNN_ACT_RELU) v = relu_f32(v);
        y[i] = __float2bfloat16_rn(v);
    }
}

// ================================================= weight gradient =============================================================
struct LinearWgradParams {
    int N, O, QC, F, nch, rows, pairs, iblocks, splits, units, stages;
    float *slots;                    // [splits][O][F] (dw itself when splits == 1)
};

template <int NW>  // accumulator columns: O rounded up to 64 (an MN-major SWIZZLE_128B operand is 64 wide)
__global__ void __launch_bounds__(LN_THREADS, 1)
k_linear_wgrad(const __grid_constant__ LinearMaps m, const LinearWgradParams p) {
    constexpr int NB = NW / 64;
    constexpr int STAGE = (2 + NB) * LN_BOX;     // [x chunk of warpgroup 0][x chunk of warpgroup 1][NB dy boxes]
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *ring = align1024(smem_dyn);
    const int NST = p.stages;
    LnCtl &S = *reinterpret_cast<LnCtl *>(ring + (size_t)NST * STAGE);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int i = 0; i < NST; ++i) { bar_init(&S.full[i], 1); bar_init(&S.empty[i], LN_CONSUMER_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == LN_CONSUMER_WARPS) {
        if (lane == 0) {
            int it = 0;
            for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
                // range-major: the units running together share their image blocks, and L2 absorbs the re-reads of dy
                const int split = u / p.pairs, pair = u % p.pairs;
                const int nx = 2 * pair + 1 < p.rows ? 2 : 1;
                for (int b = range_begin(p.iblocks, p.splits, split), b1 = range_begin(p.iblocks, p.splits, split + 1); b < b1; ++b, ++it) {
                    const int stage = it % NST;
                    bar_wait_relaxed(&S.empty[stage], ((unsigned)(it / NST) & 1u) ^ 1u, 32);
                    unsigned char *sp = ring + (size_t)stage * STAGE;
                    bar_expect_tx(&S.full[stage], (unsigned)((nx + NB) * LN_BOX));
                    for (int w = 0; w < nx; ++w) {
                        const int rb = 2 * pair + w;
                        tma_load_3d(sp + w * LN_BOX, &m.a, (rb % p.nch) * LN_KC, rb / p.nch, b * LN_M, &S.full[stage]);
                    }
                    for (int g = 0; g < NB; ++g) tma_load_2d(sp + (2 + g) * LN_BOX, &m.b, g * 64, b * LN_M, &S.full[stage]);
                }
            }
        }
        return;
    }

    const int wg = warp >> 2, wq = warp & 3;
    int it = 0;
    for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
        const int split = u / p.pairs, pair = u % p.pairs;
        const int rb = 2 * pair + wg;
        const bool live = rb < p.rows;                    // an odd number of chunks leaves warpgroup 1 one idle unit
        const int b0 = range_begin(p.iblocks, p.splits, split), b1 = range_begin(p.iblocks, p.splits, split + 1);
        float acc[NW / 2];
        for (int b = b0; b < b1; ++b, ++it) {
            const int stage = it % NST;
            bar_wait(&S.full[stage], (unsigned)(it / NST) & 1u);
            if (live) {
                const uint32_t sa = s_u32(ring + (size_t)stage * STAGE);
                const uint32_t a0 = sa + (uint32_t)(wg * LN_BOX), d0 = sa + 2u * LN_BOX;
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < 8; ++ks)             // 16 images = 16 rows of 128 bytes per instruction
                    wgmma_bf16<1, 1>(acc, gmma_desc_mn_sw128(a0 + ks * 2048, LN_BOX), gmma_desc_mn_sw128(d0 + ks * 2048, LN_BOX),
                                     (b != b0 || ks != 0) ? 1u : 0u);
                wg_commit();
            }
            if (b > b0) {
                wg_wait<1>();
                __syncwarp();
                if (lane == 0) bar_arrive(&S.empty[(it - 1) % NST]);
            }
        }
        wg_wait<0>();
        wg_hold(acc);
        __syncwarp();
        if (lane == 0) bar_arrive(&S.empty[(it - 1) % NST]);
        if (live) {
            const int prow = rb / p.nch, q0 = (rb % p.nch) * LN_KC;
            float *dst = p.slots + (size_t)split * p.O * p.F + (size_t)prow * p.QC;
#pragma unroll
            for (int i = 0; i < NW / 2; ++i) {
                const int qc = q0 + wg_row(i, wq, lane), o = wg_col(i, lane);
                if (qc < p.QC && o < p.O) dst[(size_t)o * p.F + qc] = acc[i];
            }
        }
    }
}

// ================================================= input gradient ==============================================================
struct LinearDgradParams {
    int N, QC, nch, chunks, groups, mtiles, tiles, nkc, stages, row_pitch, image_rows;
    __nv_bfloat16 *dx;
};

template <int NB>  // chunks per tile: NB * 64 accumulator columns
__global__ void __launch_bounds__(LN_THREADS, 1)
k_linear_dgrad(const __grid_constant__ LinearMaps m, const LinearDgradParams p) {
    constexpr int N = NB * 64;
    constexpr int STAGE = LN_BOX + NB * LN_WBOX;  // [dy box][NB weight boxes]
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *ring = align1024(smem_dyn);
    const int NST = p.stages;
    LnCtl &S = *reinterpret_cast<LnCtl *>(ring + (size_t)NST * STAGE);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int i = 0; i < NST; ++i) { bar_init(&S.full[i], 1); bar_init(&S.empty[i], LN_CONSUMER_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == LN_CONSUMER_WARPS) {
        if (lane == 0) {
            int it = 0;
            for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
                const int g = tile / p.mtiles, mt = tile % p.mtiles;
                for (int kc = 0; kc < p.nkc; ++kc, ++it) {
                    const int stage = it % NST;
                    bar_wait_relaxed(&S.empty[stage], ((unsigned)(it / NST) & 1u) ^ 1u, 32);
                    unsigned char *sa = ring + (size_t)stage * STAGE;
                    bar_expect_tx(&S.full[stage], (unsigned)STAGE);
                    tma_load_2d(sa, &m.a, kc * LN_KC, mt * LN_M, &S.full[stage]);
                    for (int j = 0; j < NB; ++j) {
                        // a chunk past the last one (a ragged final group) reloads the last chunk; its columns are not stored
                        const int gc = min(g * NB + j, p.chunks - 1);
                        tma_load_3d(sa + LN_BOX + j * LN_WBOX, &m.b, (gc % p.nch) * LN_KC, gc / p.nch, kc * LN_KC, &S.full[stage]);
                    }
                }
            }
        }
        return;
    }

    const int wg = warp >> 2, wq = warp & 3;
    int it = 0;
    for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
        const int g = tile / p.mtiles, mt = tile % p.mtiles;
        float acc[N / 2];
        for (int step = 0; step < p.nkc; ++step, ++it) {
            const int stage = it % NST;
            bar_wait(&S.full[stage], (unsigned)(it / NST) & 1u);
            const uint32_t a0 = s_u32(ring + (size_t)stage * STAGE) + (uint32_t)(wg * 64 * LN_KC * 2);
            const uint32_t b0 = s_u32(ring + (size_t)stage * STAGE + LN_BOX);
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < LN_KC / 16; ++ks)       // 16 outputs: 32 bytes of a dy row, 16 rows of a weight box
                wgmma_bf16<0, 1>(acc, gmma_desc_k_sw128(a0 + ks * 32), gmma_desc_mn_sw128(b0 + ks * 2048, LN_WBOX),
                                 (step | ks) != 0 ? 1u : 0u);
            wg_commit();
            if (step > 0) {
                wg_wait<1>();
                __syncwarp();
                if (lane == 0) bar_arrive(&S.empty[(it - 1) % NST]);
            }
        }
        wg_wait<0>();
        wg_hold(acc);
        __syncwarp();
        if (lane == 0) bar_arrive(&S.empty[(it - 1) % NST]);
#pragma unroll
        for (int i = 0; i < N / 2; i += 2) {              // acc[i], acc[i + 1]: columns c, c + 1 of one row
            const int n = mt * LN_M + wg * 64 + wg_row(i, wq, lane), c = wg_col(i, lane);
            const int gc = g * NB + c / 64;
            if (n >= p.N || gc >= p.chunks) continue;
            const int qc = (gc % p.nch) * LN_KC + c % 64;
            __nv_bfloat16 *dst = p.dx + ((size_t)n * p.image_rows + gc / p.nch) * p.row_pitch + qc;
            if (qc + 1 < p.QC)
                *reinterpret_cast<__nv_bfloat162 *>(dst) = __floats2bfloat162_rn(acc[i], acc[i + 1]);
            else if (qc < p.QC)
                *dst = __float2bfloat16_rn(acc[i]);
        }
    }
}

// dense [N][O] -> [N][O8] with zero columns, the 16-byte row stride a TMA map needs
__global__ void __launch_bounds__(256) k_linear_pad_rows(const __nv_bfloat16 *__restrict__ src, __nv_bfloat16 *__restrict__ dst, long N,
                                                         int O, int O8) {
    const long total = N * O8;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const long n = i / O8;
        const int o = (int)(i % O8);
        dst[i] = o < O ? src[n * O + o] : __float2bfloat16_rn(0.0f);
    }
}

// ================================================= softmax cross-entropy ========================================================
// One warp per row, lane t holds logits t, t + 32, ... (O <= 256: 8 each), all read before anything is written (in place).
// SOFT: the target q_t of pcnn_softmax_ce_soft_bf16, built in fp32 from the labels, labels_b and the weights of SoftTarget.
struct SoftTarget {
    const uint8_t *labels_b;  // NULL: m_t = [t == label]
    float lam, oml;           // RN32(lam), RN32(1 - lam)
    float ome, eps_o;         // RN32(1 - eps), RN32(eps / O)
    const int *count;         // PIXELS: the non-ignored rows, counted by k_count_targets
    int ignore;               // PIXELS: the ignored target, -1 for none
};

// PIXELS (hard target only): pcnn_softmax_ce_pixels_bf16.  The scale is RN32(1 / count) read from the device; a row whose target is
// st.ignore gets dlogits +0 and loss 0; every other row is exactly the hard call's at that scale.
template <bool SOFT, bool PIXELS = false>
__global__ void __launch_bounds__(256) k_softmax_ce_bf16(const __nv_bfloat16 *z, const uint8_t *__restrict__ labels, int N, int O,
                                                         double scale, __nv_bfloat16 *d, float *__restrict__ loss, int *__restrict__ pred,
                                                         const SoftTarget st) {
    const int lane = threadIdx.x & 31;
    const long warp = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5;
    const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
    for (long r = warp; r < N; r += nwarps) {
        float v[8];
        bool nan = false;
        float best = -INFINITY;
        int bi = O;                                       // first index of the largest logit (O: none yet)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int t = lane + 32 * j;
            v[j] = t < O ? __bfloat162float(z[r * O + t]) : -INFINITY;
            if (t < O) {
                nan |= isnan(v[j]);
                if (bi == O || v[j] > best) { best = v[j]; bi = t; }
            }
        }
        for (int s = 16; s; s >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, s);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, s);
            if (oi < O && (bi == O || ob > best || (ob == best && oi < bi))) { best = ob; bi = oi; }
        }
        nan = __any_sync(0xffffffffu, nan);
        double mx = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (lane + 32 * j < O) mx = fmax(mx, (double)v[j]);
        for (int s = 16; s; s >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, s));
        double den = 0.0;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (lane + 32 * j < O) den += exp((double)v[j] - mx);
        for (int s = 16; s; s >>= 1) den += __shfl_xor_sync(0xffffffffu, den, s);
        const int y = labels[r];
        if constexpr (PIXELS) {
            if (y == st.ignore) {
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    if (lane + 32 * j < O) d[r * O + lane + 32 * j] = __float2bfloat16_rn(0.0f);
                if (lane == 0) {
                    if (loss) loss[r] = 0.0f;
                    if (pred) pred[r] = nan ? -1 : bi;
                }
                continue;
            }
            scale = (double)(float)(1.0 / (double)*st.count);
        }
        if constexpr (!SOFT) {
            const bool bad = nan || y >= O;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int t = lane + 32 * j;
                if (t >= O) continue;
                const double g = (exp((double)v[j] - mx) / den - (t == y ? 1.0 : 0.0)) * scale;
                d[r * O + t] = bad ? __float2bfloat16_rn(NAN) : __float2bfloat16_rn((float)g);
                if (t == y && loss) loss[r] = nan ? NAN : (float)(-(((double)v[j] - mx) - log(den)));
            }
            if (lane == 0) {
                if (loss && y >= O) loss[r] = NAN;
                if (pred) pred[r] = nan ? -1 : bi;
            }
        } else {
            const int yb = st.labels_b ? st.labels_b[r] : y;
            const bool bad = nan || y >= O || yb >= O;
            const double lden = log(den);
            double part = 0.0;                            // this lane's terms of sum q_t ((z_t - m) - log den)
            int terms = 0;
            bool hot = false;                             // this lane holds a q_t == 1
            float lhot = 0.0f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int t = lane + 32 * j;
                if (t >= O) continue;
                // m_t = RN(RN([t == yb] (1 - lam)) + RN([t == y] lam)), or [t == y] without labels_b; q_t = RN(RN(m_t (1 - eps)) + eps / O)
                const float mt = st.labels_b ? __fadd_rn(t == yb ? st.oml : 0.0f, t == y ? st.lam : 0.0f) : (t == y ? 1.0f : 0.0f);
                const float q = __fadd_rn(__fmul_rn(mt, st.ome), st.eps_o);
                const double g = (exp((double)v[j] - mx) / den - (double)q) * scale;
                d[r * O + t] = bad ? __float2bfloat16_rn(NAN) : __float2bfloat16_rn((float)g);
                if (q != 0.0f) {                          // terms with q_t = 0 skipped
                    part += (double)q * (((double)v[j] - mx) - lden);
                    ++terms;
                    if (q == 1.0f) {
                        hot = true;
                        lhot = (float)(-(((double)v[j] - mx) - lden));
                    }
                }
            }
            for (int s = 16; s; s >>= 1) {
                part += __shfl_xor_sync(0xffffffffu, part, s);
                terms += __shfl_xor_sync(0xffffffffu, terms, s);
            }
            // a one-hot target takes the hard kernel's expression, so that its loss bits (NaN ones from +-Inf logits included) match
            const bool one_hot = terms == 1 && __any_sync(0xffffffffu, hot);
            if (loss && (one_hot ? hot : lane == 0)) loss[r] = bad ? NAN : one_hot ? lhot : (float)(-part);
            if (lane == 0 && pred) pred[r] = nan ? -1 : bi;
        }
    }
}

// count[0] = the targets that are not `ignore` (-1: all): per-CTA counts added with integer atomics, which are exact in any order
__global__ void __launch_bounds__(256) k_count_targets(const uint8_t *__restrict__ t, long n, int ignore, int *count) {
    int c = 0;
    for (long i = blockIdx.x * 256L + threadIdx.x; i < n; i += (long)gridDim.x * 256) c += (int)t[i] != ignore;
    for (int s = 16; s; s >>= 1) c += __shfl_xor_sync(0xffffffffu, c, s);
    __shared__ int part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int sum = 0;
        for (int w = 0; w < 8; ++w) sum += part[w];
        atomicAdd(count, sum);
    }
}

}  // namespace

// ================================================= host ==========================================================================
struct LinearShape {
    int N, P, Q, C, O, QC, F, row_pitch, image_rows, nch, wpitch;
    int mtiles, fsteps, fsplits, funits, npad, fstages;
    int wrows, wpairs, wsplits, wunits, wn, wstages;
    int dchunks, dnb, dgroups, dtiles, nkc, dstages;
};

static int cap_stages(size_t stage_bytes) {
    const int n = (int)(((size_t)LN_SMEM_BUDGET - sizeof(LnCtl) - 1024) / stage_bytes);
    return n > LN_MAX_STAGES ? LN_MAX_STAGES : n;
}
static size_t fwd_stage(int npad) { return (size_t)LN_BOX + (size_t)npad * LN_KC * 2; }
static size_t wgrad_stage(int wn) { return (size_t)(2 + wn / 64) * LN_BOX; }
static size_t dgrad_stage(int nb) { return (size_t)LN_BOX + (size_t)nb * LN_WBOX; }
static size_t smem_for(size_t stage_bytes, int stages) { return (size_t)stages * stage_bytes + sizeof(LnCtl) + 1024; }

// the domain of pcnn_linear_plan_create (its refusals name that call) and every tiling decision: a function of the shape only
static int linear_shape(int N, int P, int Q, int C, int O, int row_pitch, int image_rows, LinearShape *s) {
    const char *fn = "pcnn_linear_plan_create";
    PCNN_REQUIRE(N >= 1 && P >= 1 && Q >= 1 && C >= 1 && O >= 1 && O <= 256, PCNN_ERR_ARG,
                 "%s: bad shape N=%d P=%d Q=%d C=%d O=%d: N, P, Q, C >= 1 and 1 <= O <= 256 are required", fn, N, P, Q, C, O);
    const long long F = (long long)P * Q * C;
    PCNN_REQUIRE(F <= LN_MAX_F, PCNN_ERR_ARG, "%s: F = P*Q*C = %lld features: at most 2^24 = %lld are supported", fn, F, LN_MAX_F);
    const int QC = Q * C;
    if (row_pitch == 0) row_pitch = (QC + 7) / 8 * 8;
    PCNN_REQUIRE(row_pitch >= QC && row_pitch % 8 == 0, PCNN_ERR_ARG,
                 "%s: row pitch %d must be >= Q*C = %d and a multiple of 8 elements (TMA 16-byte strides); so a hidden width that "
                 "feeds another linear layer (P = Q = 1, C = O, row_pitch = O) must be a multiple of 8", fn, row_pitch, QC);
    if (image_rows == 0) image_rows = P;
    PCNN_REQUIRE(image_rows >= P, PCNN_ERR_ARG, "%s: image pitch of %d rows is smaller than P = %d", fn, image_rows, P);
    s->N = N; s->P = P; s->Q = Q; s->C = C; s->O = O; s->QC = QC; s->F = (int)F;
    s->row_pitch = row_pitch; s->image_rows = image_rows;
    s->nch = (QC + LN_KC - 1) / LN_KC;
    s->wpitch = (QC + 7) / 8 * 8;
    s->mtiles = (int)(((long long)N + LN_M - 1) / LN_M);
    s->fsteps = P * s->nch;
    const int want_f = (LN_TARGET_UNITS + s->mtiles - 1) / s->mtiles, most_f = s->fsteps / LN_MIN_SPLIT_STEPS;
    s->fsplits = want_f < most_f ? want_f : most_f;
    if (s->fsplits < 1) s->fsplits = 1;
    s->npad = (O + 15) / 16 * 16;
    s->fstages = cap_stages(fwd_stage(s->npad));
    s->wrows = s->fsteps;
    s->wpairs = (s->wrows + 1) / 2;
    const int want_w = (LN_TARGET_UNITS + s->wpairs - 1) / s->wpairs;
    s->wsplits = want_w < s->mtiles ? want_w : s->mtiles;
    s->wn = (O + 63) / 64 * 64;
    s->wstages = cap_stages(wgrad_stage(s->wn));
    s->dchunks = s->fsteps;
    s->dnb = s->dchunks < LN_DGRAD_MAX_BOXES ? s->dchunks : LN_DGRAD_MAX_BOXES;
    s->dgroups = (s->dchunks + s->dnb - 1) / s->dnb;
    s->nkc = (O + LN_KC - 1) / LN_KC;
    s->dstages = cap_stages(dgrad_stage(s->dnb));
    const long long funits = (long long)s->mtiles * s->fsplits, wunits = (long long)s->wpairs * s->wsplits,
                    dtiles = (long long)s->mtiles * s->dgroups;
    PCNN_REQUIRE(funits < (1LL << 31) && wunits < (1LL << 31) && dtiles < (1LL << 31), PCNN_ERR_ARG,
                 "%s: N = %d images with F = %lld features: the work units exceed the int range", fn, N, F);
    s->funits = (int)funits; s->wunits = (int)wunits; s->dtiles = (int)dtiles;
    return PCNN_OK;
}

// a plan of pcnn_linear_plan_create: w is [O][P][wpitch], rows of Q*C in-row elements; the pad columns are zeroed at creation and
// nothing writes them again
struct LinearPlan : pcnn_conv_plan {
    static constexpr const char *made_by = "pcnn_linear_plan_create";
    LinearShape sh;
    int act;
    CUtensorMap map_w_fwd;           // {QC, P, O}, box {64, 1, npad}: K-major B of the forward
    CUtensorMap map_w_dgrad;         // the same tensor, box {64, 1, 64}: MN-major B of the input gradient
    int fwd(pcnn_ctx *ctx, const void *x_bf16, void *y_bf16) override;
};

typedef void (*linear_fn)(const LinearMaps, const LinearFwdParams);
typedef void (*wgrad_fn)(const LinearMaps, const LinearWgradParams);
typedef void (*dgrad_fn)(const LinearMaps, const LinearDgradParams);
static const void *fwd_variant(int npad) {
    static const linear_fn t[16] = {k_linear_fwd<16>,  k_linear_fwd<32>,  k_linear_fwd<48>,  k_linear_fwd<64>,
                                    k_linear_fwd<80>,  k_linear_fwd<96>,  k_linear_fwd<112>, k_linear_fwd<128>,
                                    k_linear_fwd<144>, k_linear_fwd<160>, k_linear_fwd<176>, k_linear_fwd<192>,
                                    k_linear_fwd<208>, k_linear_fwd<224>, k_linear_fwd<240>, k_linear_fwd<256>};
    return reinterpret_cast<const void *>(t[npad / 16 - 1]);
}
static const void *wgrad_variant(int wn) {
    static const wgrad_fn t[4] = {k_linear_wgrad<64>, k_linear_wgrad<128>, k_linear_wgrad<192>, k_linear_wgrad<256>};
    return reinterpret_cast<const void *>(t[wn / 64 - 1]);
}
static const void *dgrad_variant(int nb) {
    static const dgrad_fn t[4] = {k_linear_dgrad<1>, k_linear_dgrad<2>, k_linear_dgrad<3>, k_linear_dgrad<4>};
    return reinterpret_cast<const void *>(t[nb - 1]);
}

static int configure(pcnn_ctx *ctx) {
    static bool configured[64] = {};        // function attributes are per device
    if (configured[ctx->device & 63]) return PCNN_OK;
    for (int v = 1; v <= 16; ++v)
        PCNN_CUDA(cudaFuncSetAttribute(fwd_variant(16 * v), cudaFuncAttributeMaxDynamicSharedMemorySize, LN_SMEM_BUDGET + 2048));
    for (int v = 1; v <= 4; ++v) {
        PCNN_CUDA(cudaFuncSetAttribute(wgrad_variant(64 * v), cudaFuncAttributeMaxDynamicSharedMemorySize, LN_SMEM_BUDGET + 2048));
        PCNN_CUDA(cudaFuncSetAttribute(dgrad_variant(v), cudaFuncAttributeMaxDynamicSharedMemorySize, LN_SMEM_BUDGET + 2048));
    }
    configured[ctx->device & 63] = true;
    return PCNN_OK;
}

// x viewed as {Q*C, P, N}: the extents stop at the row's features and the image's rows, so pad is never read
static int x_map(CUtensorMap *map, const void *x, const LinearShape &s) {
    const uint64_t dims[3] = {(uint64_t)s.QC, (uint64_t)s.P, (uint64_t)s.N};
    const uint64_t str[2] = {(uint64_t)s.row_pitch * 2, (uint64_t)s.image_rows * s.row_pitch * 2};
    const uint32_t box[3] = {LN_KC, 1, LN_M};
    return make_map_bf16(map, const_cast<void *>(x), 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

// dy [N][O] as a map {O, N} with box {64, 128}; rows of O % 8 != 0 elements go through a zero-padded copy at `pad_buf`
static int dy_map(pcnn_ctx *ctx, CUtensorMap *map, const void *dy, void *pad_buf, const LinearShape &s) {
    const int O8 = (s.O + 7) / 8 * 8;
    const void *src = dy;
    if (O8 != s.O) {
        const long total = (long)s.N * O8;
        long blocks = (total + 255) / 256;
        if (blocks > (long)ctx->sm_count * 8) blocks = (long)ctx->sm_count * 8;
        k_linear_pad_rows<<<(int)blocks, 256, 0, ctx->stream>>>(static_cast<const __nv_bfloat16 *>(dy), static_cast<__nv_bfloat16 *>(pad_buf),
                                                                s.N, s.O, O8);
        PCNN_CHECK_LAUNCH(ctx);
        src = pad_buf;
    }
    const uint64_t dims[2] = {(uint64_t)s.O, (uint64_t)s.N};
    const uint64_t str[1] = {(uint64_t)O8 * 2};
    const uint32_t box[2] = {LN_KC, LN_M};
    return make_map_bf16(map, const_cast<void *>(src), 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

static size_t dy_pad_bytes(const LinearShape &s) {
    return s.O % 8 ? ((size_t)s.N * ((s.O + 7) / 8 * 8) * 2 + 255) / 256 * 256 : 0;
}

extern "C" int pcnn_linear_info(int N, int P, int Q, int C, int O, int row_pitch, int image_rows, int *out12) {
    PCNN_REQUIRE(out12, PCNN_ERR_ARG, "pcnn_linear_info: NULL argument");
    LinearShape s;
    int rc = linear_shape(N, P, Q, C, O, row_pitch, image_rows, &s);
    if (rc) return rc;
    const int v[12] = {s.row_pitch, s.mtiles, s.fsteps, s.fsplits, s.fstages, s.wpairs, s.wsplits, s.wstages,
                       s.dtiles, s.dnb, s.dstages, s.npad};
    memcpy(out12, v, sizeof(v));
    return PCNN_OK;
}

extern "C" int pcnn_linear_plan_create(pcnn_ctx *ctx, int N, int P, int Q, int C, int O, int row_pitch, int image_rows, int act,
                                       const float *w_host, const float *b_host, pcnn_conv_plan **out) {
    const char *fn = "pcnn_linear_plan_create";
    PCNN_REQUIRE(ctx && w_host && out, PCNN_ERR_ARG, "%s: NULL argument", fn);
    PCNN_REQUIRE_ACT(fn, act);
    LinearShape s;
    int rc = linear_shape(N, P, Q, C, O, row_pitch, image_rows, &s);
    if (rc) return rc;
    pcnn_device_guard g(ctx->device);
    if ((rc = configure(ctx))) return rc;
    std::unique_ptr<LinearPlan> pl(new LinearPlan());   // frees a half-built plan on every early return below
    pl->sh = s;
    pl->act = act;
    pl->cols = s.QC; pl->pitch = s.wpitch;
    pl->n = (long long)O * s.F;
    pl->K = O;
    if ((rc = pcnn_plan_upload(ctx, pl.get(), &pl->w, (size_t)O * P * s.wpitch * 2, w_host, b_host))) return rc;
    const uint64_t dims[3] = {(uint64_t)s.QC, (uint64_t)P, (uint64_t)O};
    const uint64_t str[2] = {(uint64_t)s.wpitch * 2, (uint64_t)P * s.wpitch * 2};
    const uint32_t box_f[3] = {LN_KC, 1, (uint32_t)s.npad}, box_d[3] = {LN_KC, 1, 64};
    if ((rc = make_map_bf16(&pl->map_w_fwd, pl->w, 3, dims, str, box_f, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B)))
        return rc;
    if ((rc = make_map_bf16(&pl->map_w_dgrad, pl->w, 3, dims, str, box_d, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B)))
        return rc;
    *out = pl.release();
    return PCNN_OK;
}

int LinearPlan::fwd(pcnn_ctx *ctx, const void *x_bf16, void *y_bf16) {
    PCNN_REQUIRE(((uintptr_t)y_bf16 & 15) == 0, PCNN_ERR_ARG, "pcnn_conv_tc_fwd: the output must be 16-byte aligned");
    const LinearShape &s = sh;
    LinearMaps m;
    memset(&m, 0, sizeof(m));
    int rc = x_map(&m.a, x_bf16, s);
    if (rc) return rc;
    m.b = map_w_fwd;
    LinearFwdParams p;
    p.N = s.N; p.O = s.O; p.nch = s.nch; p.steps = s.fsteps; p.splits = s.fsplits; p.mtiles = s.mtiles; p.units = s.funits;
    p.stages = s.fstages; p.act = act; p.bias = bias;
    p.y = static_cast<__nv_bfloat16 *>(y_bf16);
    p.slots = nullptr;
    const long total = (long)s.N * s.O;
    if (s.fsplits > 1 && (rc = pcnn_scratch(ctx, (size_t)s.fsplits * total * sizeof(float), (void **)&p.slots))) return rc;
    const int grid = p.units < ctx->sm_count ? p.units : ctx->sm_count;
    void *args[] = {&m, &p};
    PCNN_CUDA(cudaLaunchKernel(fwd_variant(s.npad), dim3((unsigned)grid), dim3(LN_THREADS), args, smem_for(fwd_stage(s.npad), s.fstages),
                               ctx->stream));
    PCNN_CHECK_LAUNCH(ctx);
    if (s.fsplits > 1) {
        long blocks = (total + 255) / 256;
        if (blocks > (long)ctx->sm_count * 8) blocks = (long)ctx->sm_count * 8;
        k_linear_fwd_reduce<<<(int)blocks, 256, 0, ctx->stream>>>(p.slots, s.fsplits, bias, act, p.y, total, s.O);
        PCNN_CHECK_LAUNCH(ctx);
    }
    return PCNN_OK;
}

extern "C" int pcnn_linear_wgrad(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *x_bf16, const void *dy_bf16, float *dw_f32) {
    const char *fn = "pcnn_linear_wgrad";
    PCNN_REQUIRE(ctx && plan && x_bf16 && dy_bf16 && dw_f32, PCNN_ERR_ARG, "%s: NULL argument", fn);
    LinearPlan *pl;
    int rc = plan_as(fn, plan, &pl);
    if (rc) return rc;
    PCNN_REQUIRE(((uintptr_t)x_bf16 & 15) == 0 && ((uintptr_t)dy_bf16 & 15) == 0 && ((uintptr_t)dw_f32 & 15) == 0, PCNN_ERR_ARG,
                 "%s: x, dy and dw must be 16-byte aligned", fn);
    const LinearShape &s = pl->sh;
    pcnn_device_guard g(ctx->device);
    const size_t pad = dy_pad_bytes(s), nout = (size_t)s.O * s.F;
    unsigned char *scratch = nullptr;
    const size_t need = pad + (s.wsplits > 1 ? (size_t)s.wsplits * nout * sizeof(float) : 0);
    if (need && (rc = pcnn_scratch(ctx, need, (void **)&scratch))) return rc;
    LinearMaps m;
    memset(&m, 0, sizeof(m));
    if ((rc = x_map(&m.a, x_bf16, s))) return rc;
    if ((rc = dy_map(ctx, &m.b, dy_bf16, scratch, s))) return rc;
    LinearWgradParams p;
    p.N = s.N; p.O = s.O; p.QC = s.QC; p.F = s.F; p.nch = s.nch; p.rows = s.wrows; p.pairs = s.wpairs; p.iblocks = s.mtiles;
    p.splits = s.wsplits; p.units = s.wunits; p.stages = s.wstages;
    p.slots = s.wsplits > 1 ? reinterpret_cast<float *>(scratch + pad) : dw_f32;
    const int grid = p.units < ctx->sm_count ? p.units : ctx->sm_count;
    void *args[] = {&m, &p};
    PCNN_CUDA(cudaLaunchKernel(wgrad_variant(s.wn), dim3((unsigned)grid), dim3(LN_THREADS), args, smem_for(wgrad_stage(s.wn), s.wstages),
                               ctx->stream));
    PCNN_CHECK_LAUNCH(ctx);
    return s.wsplits > 1 ? pcnn_conv_wgrad_reduce_slots(ctx, p.slots, dw_f32, s.wsplits, (int)nout) : PCNN_OK;
}

extern "C" int pcnn_linear_dgrad(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *dy_bf16, void *dx_bf16) {
    const char *fn = "pcnn_linear_dgrad";
    PCNN_REQUIRE(ctx && plan && dy_bf16 && dx_bf16, PCNN_ERR_ARG, "%s: NULL argument", fn);
    LinearPlan *pl;
    int rc = plan_as(fn, plan, &pl);
    if (rc) return rc;
    PCNN_REQUIRE(((uintptr_t)dy_bf16 & 15) == 0 && ((uintptr_t)dx_bf16 & 15) == 0, PCNN_ERR_ARG, "%s: dy and dx must be 16-byte aligned",
                 fn);
    const LinearShape &s = pl->sh;
    pcnn_device_guard g(ctx->device);
    unsigned char *scratch = nullptr;
    if (dy_pad_bytes(s) && (rc = pcnn_scratch(ctx, dy_pad_bytes(s), (void **)&scratch))) return rc;
    LinearMaps m;
    memset(&m, 0, sizeof(m));
    if ((rc = dy_map(ctx, &m.a, dy_bf16, scratch, s))) return rc;
    m.b = pl->map_w_dgrad;
    LinearDgradParams p;
    p.N = s.N; p.QC = s.QC; p.nch = s.nch; p.chunks = s.dchunks; p.groups = s.dgroups; p.mtiles = s.mtiles; p.tiles = s.dtiles;
    p.nkc = s.nkc; p.stages = s.dstages; p.row_pitch = s.row_pitch; p.image_rows = s.image_rows;
    p.dx = static_cast<__nv_bfloat16 *>(dx_bf16);
    const int grid = p.tiles < ctx->sm_count ? p.tiles : ctx->sm_count;
    void *args[] = {&m, &p};
    PCNN_CUDA(cudaLaunchKernel(dgrad_variant(s.dnb), dim3((unsigned)grid), dim3(LN_THREADS), args, smem_for(dgrad_stage(s.dnb), s.dstages),
                               ctx->stream));
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_softmax_ce_bf16(pcnn_ctx *ctx, const void *logits_bf16, const uint8_t *labels, int N, int O, float scale,
                                    void *dlogits_bf16, float *loss_f32, int *pred_i32) {
    const char *fn = "pcnn_softmax_ce_bf16";
    PCNN_REQUIRE(ctx && logits_bf16 && labels && dlogits_bf16, PCNN_ERR_ARG, "%s: NULL context, logits, labels or dlogits", fn);
    PCNN_REQUIRE(N >= 1 && O >= 1 && O <= 256, PCNN_ERR_ARG, "%s: N = %d, O = %d: N >= 1 and 1 <= O <= 256 are required", fn, N, O);
    const size_t zb = (size_t)N * O * 2;
    const uintptr_t z = (uintptr_t)logits_bf16, d = (uintptr_t)dlogits_bf16;
    PCNN_REQUIRE(d == z || d + zb <= z || z + zb <= d, PCNN_ERR_ARG, "%s: dlogits overlaps logits without being the same buffer", fn);
    pcnn_device_guard g(ctx->device);
    long blocks = ((long)N * 32 + 255) / 256;
    if (blocks > (long)ctx->sm_count * 8) blocks = (long)ctx->sm_count * 8;
    k_softmax_ce_bf16<false><<<(int)blocks, 256, 0, ctx->stream>>>(static_cast<const __nv_bfloat16 *>(logits_bf16), labels, N, O,
                                                                   (double)scale, static_cast<__nv_bfloat16 *>(dlogits_bf16), loss_f32,
                                                                   pred_i32, SoftTarget{});
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_softmax_ce_soft_bf16(pcnn_ctx *ctx, const void *logits_bf16, const uint8_t *labels, const uint8_t *labels_b, double lam,
                                         double smoothing, int N, int O, float scale, void *dlogits_bf16, float *loss_f32, int *pred_i32) {
    const char *fn = "pcnn_softmax_ce_soft_bf16";
    PCNN_REQUIRE(ctx && logits_bf16 && labels && dlogits_bf16, PCNN_ERR_ARG, "%s: NULL context, logits, labels or dlogits", fn);
    PCNN_REQUIRE(N >= 1 && O >= 1 && O <= 256, PCNN_ERR_ARG, "%s: N = %d, O = %d: N >= 1 and 1 <= O <= 256 are required", fn, N, O);
    PCNN_REQUIRE(std::isfinite(lam) && lam >= 0.0 && lam <= 1.0, PCNN_ERR_ARG, "%s: lam = %g: a finite 0 <= lam <= 1 is required", fn, lam);
    PCNN_REQUIRE(smoothing >= 0.0 && smoothing <= 1.0, PCNN_ERR_ARG, "%s: smoothing = %g: 0 <= smoothing <= 1 is required", fn, smoothing);
    const size_t zb = (size_t)N * O * 2;
    const uintptr_t z = (uintptr_t)logits_bf16, d = (uintptr_t)dlogits_bf16;
    PCNN_REQUIRE(d == z || d + zb <= z || z + zb <= d, PCNN_ERR_ARG, "%s: dlogits overlaps logits without being the same buffer", fn);
    SoftTarget st;
    st.labels_b = labels_b;
    st.lam = (float)lam;
    st.oml = (float)(1.0 - lam);
    st.ome = (float)(1.0 - smoothing);
    st.eps_o = (float)(smoothing / O);
    pcnn_device_guard g(ctx->device);
    long blocks = ((long)N * 32 + 255) / 256;
    if (blocks > (long)ctx->sm_count * 8) blocks = (long)ctx->sm_count * 8;
    k_softmax_ce_bf16<true><<<(int)blocks, 256, 0, ctx->stream>>>(static_cast<const __nv_bfloat16 *>(logits_bf16), labels, N, O,
                                                                  (double)scale, static_cast<__nv_bfloat16 *>(dlogits_bf16), loss_f32,
                                                                  pred_i32, st);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_softmax_ce_pixels_bf16(pcnn_ctx *ctx, const void *logits_bf16, const uint8_t *targets, int pixels, int O, int ignore_index,
                                           void *dlogits_bf16, float *loss_f32, int *pred_i32, int *count_i32) {
    const char *fn = "pcnn_softmax_ce_pixels_bf16";
    PCNN_REQUIRE(ctx && logits_bf16 && targets && dlogits_bf16 && count_i32, PCNN_ERR_ARG,
                 "%s: NULL context, logits, targets, dlogits or count (only loss and pred may be NULL)", fn);
    PCNN_REQUIRE(pixels >= 1 && O >= 1 && O <= 256, PCNN_ERR_ARG, "%s: pixels = %d, O = %d: pixels >= 1 and 1 <= O <= 256 are required", fn,
                 pixels, O);
    PCNN_REQUIRE(ignore_index >= -1 && ignore_index <= 255, PCNN_ERR_ARG, "%s: ignore_index = %d: -1 (none) or 0 .. 255 is required", fn,
                 ignore_index);
    const size_t zb = (size_t)pixels * O * 2;
    const uintptr_t z = (uintptr_t)logits_bf16, d = (uintptr_t)dlogits_bf16;
    PCNN_REQUIRE(d == z || d + zb <= z || z + zb <= d, PCNN_ERR_ARG, "%s: dlogits overlaps logits without being the same buffer", fn);
    pcnn_device_guard g(ctx->device);
    PCNN_CUDA(cudaMemsetAsync(count_i32, 0, sizeof(int), ctx->stream));
    long cblocks = ((long)pixels + 255) / 256;
    if (cblocks > (long)ctx->sm_count * 4) cblocks = (long)ctx->sm_count * 4;
    k_count_targets<<<(int)cblocks, 256, 0, ctx->stream>>>(targets, pixels, ignore_index, count_i32);
    PCNN_CHECK_LAUNCH(ctx);
    SoftTarget st{};
    st.count = count_i32;
    st.ignore = ignore_index;
    long blocks = ((long)pixels * 32 + 255) / 256;
    if (blocks > (long)ctx->sm_count * 8) blocks = (long)ctx->sm_count * 8;
    k_softmax_ce_bf16<false, true><<<(int)blocks, 256, 0, ctx->stream>>>(static_cast<const __nv_bfloat16 *>(logits_bf16), targets, pixels, O,
                                                                         0.0, static_cast<__nv_bfloat16 *>(dlogits_bf16), loss_f32,
                                                                         pred_i32, st);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
