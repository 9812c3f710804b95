// parallel-cnn_b200/csrc/conv_wide_bwd_tc.cu -- weight and input gradients of the wide-channel forward (conv_wide_tc.cu) on the
// Hopper tensor cores: pcnn_conv_wide_wgrad, pcnn_conv_wide_dgrad and the host-only query pcnn_conv_wide_bwd_info.  Same
// domain, pitches and pad rules as pcnn_conv_wide_plan_create; dy is dense [N][P][Q][K] as that forward writes it.
//
// Weight gradient, a GEMM over pixels:  dw[(r, s, c)][k] = sum_{n,p,q} x[n][p*st + r][q*st + s][c] * dy[n][p][q][k].
//   * Rows: R*S*ceil(C/64) row blocks of 64, one (tap, 64-channel chunk) each.  A work unit is a pair of row blocks (one per
//     consumer warpgroup, M = 64 each) and a range of the forward's Pt x Qt = 128 pixel blocks; the reduction runs over the
//     range, 16 pixels per m64nNk16.  Columns: the filters rounded up to 64 (N = 64 .. 256).
//   * A: the x box {64 channels, Qt, Pt, 1} of the forward's per-phase map at (q0 + s/st, p0 + r/st): 128 pixel rows of 64
//     channels, i.e. MN-major with SWIZZLE_128B.  B: a box {64 filters, Qt, Pt, 1} of a dense map of dy, MN-major the same
//     way; both warpgroups read the same dy boxes.  TMA zero-fills dy pixels past P / Q and filters >= K, so ragged blocks
//     need no masks, and x never reads pad (its extents end at the image).
//   * Units are ordered range-major: the CTAs running at the same time share a pixel range and L2 absorbs the re-reads of dy.
//   * Each unit writes its two row blocks as a partial dw (KRSC, channels < C, filters < K) into the slot of its range; a
//     second kernel adds the slots in a fixed order (deterministic, no atomics, as conv_wgrad_tc.cu).
//
// Input gradient, one stride-1 "full" correlation per phase (a, b) = (h mod st, w mod st) of dx:
//     dx[n][st*u + a][st*v + b][c] = sum_{i,j} sum_k dy[n][u - i][v - j][k] * f[k][a + st*i][b + st*j][c]
//   over i < ceil((R - a)/st), j < ceil((S - b)/st).
//   * A tile is (phase, Pt x Qt = 128 block of the phase's grid, image, channel group of <= 256); the reduction runs over
//     (i, j, 64-filter chunk).  A: the dy box {64 filters, Qt, Pt, 1} at (v0 - j, u0 - i), K-major; the signed coordinates
//     zero-fill dy above / left of the image as well as past P / Q, so no padded copy of dy exists.  B: the filters as bf16
//     [R*S][C][K] (one conversion kernel into scratch), a box {64 filters, N channels, 1 tap}, K-major; TMA zero-fills
//     filters >= K and channels >= C.
//   * Epilogue as the forward's (bf16 staging tile per warpgroup, TMA store), through one map of dx per phase: base
//     a * row_pitch + b * C, strides st*C, st*row_pitch, image_rows*row_pitch, extents ceil((W-b)/st), ceil((H-a)/st).  The
//     stores clip there, so pad and the other phases are never written; rows and columns no window covers come out as
//     written zeros.  A phase without taps (st > R or st > S) writes its tiles from accumulators zeroed explicitly.
//
// Zero padding (the _padded entry points) changes box coordinates only.  Weight gradient: x through the forward's per-tap phase
// and offset (ConvWideTaps).  Input gradient: the tiles and dx maps stay those of the unpadded phases (a, b) of dx; with
// a + pad_h = st * off_h + rho_h, phase a takes the taps r = rho_h + st*i (none when rho_h >= R) and reads dy at row u - i + off_h,
// columns the same with pad_w.  At pad 0, rho_h = a and off_h = 0.
//
// Dilation (the _dilated entry points).  Weight gradient: the forward's tap table, device code unchanged.  Input gradient: tap r
// reaches dx row st*u + a when r*dil_h = a + pad_h (mod st).  With g = gcd(dil_h, st), phase a has no taps unless g divides
// a + pad_h; then its taps are r = rho_h + (st/g)*i (rho_h the least such r, none when rho_h >= R) and tap i reads dy row
// u - (dil_h/g)*i + off_h with off_h = (a + pad_h - rho_h*dil_h)/st, exact.  Columns the same with dil_w and pad_w.  The tap step
// st/g and the dy step dil_h/g are parameters of the producer's addresses only; at dilation 1 they are st and 1.
//
// Warp roles (288 threads, 1 CTA/SM, persistent): warps 0-7 = two consumer warpgroups, warp 8 = TMA producer.
#include "tc_common.cuh"

#include <cuda_bf16.h>

#include <numeric>
#include <type_traits>

using namespace pcnn_tc;

namespace {

constexpr int WB_THREADS = 288;
constexpr int WB_CONSUMER_WARPS = 8;
constexpr int WB_KC = 64;                        // channels / filters per 128-byte SWIZZLE_128B row
constexpr int WB_BOX_BYTES = 128 * WB_KC * 2;    // 128 pixels x 64 channels: 16 KB
constexpr int WB_STG_BYTES = 64 * WB_KC * 2;     // one staging sub-tile of the input gradient: 64 pixels x 64 channels
constexpr int WB_MAX_STAGES = 8;
constexpr int WB_SMEM_BUDGET = 225 * 1024;
constexpr int WB_BLOCKS_PER_SPLIT = 32;          // pixel blocks per weight-gradient range (at least, when there are 32)
constexpr int WB_MAX_GROUP = 256;                // channels per input-gradient tile (the widest wgmma)

struct WideCtl {
    unsigned long long full[WB_MAX_STAGES], empty[WB_MAX_STAGES];
};

__device__ __forceinline__ unsigned char *align1024(unsigned char *p) {
    return reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(p) + 1023) & ~(uintptr_t)1023);
}

// ================================================= weight gradient ======================================================
struct WideWgradParams {
    int Pt, Qt, n_pb, n_qb;          // the forward's pixel block and blocks per image column / row
    int R, S, stride, nch, C, K;
    int rows, pairs;                 // row blocks R*S*nch, pairs of them (units per pixel range)
    int blocks, splits, units;       // pixel blocks N*n_pb*n_qb, pixel ranges, pairs * splits
    int stages;
    float *slots;                    // [splits][K][R][S][C]
    ConvWideTaps taps;               // the forward's x phase and box offset of every tap row / column
};

struct WideWgradMaps {
    CUtensorMap x[16];               // the forward's phase maps of x
    CUtensorMap dy;                  // {K, Q, P, N}, box {64, Qt, Pt, 1}
};

__host__ __device__ __forceinline__ int split_begin(const WideWgradParams &p, int split) {
    return (int)((long long)split * p.blocks / p.splits);
}

template <int N>   // accumulator columns: the filters rounded up to 64 (an MN-major SWIZZLE_128B operand is 64 wide)
__global__ void __launch_bounds__(WB_THREADS, 1)
k_conv_wide_wgrad(const __grid_constant__ WideWgradMaps m, const WideWgradParams p) {
    constexpr int NB = N / 64;
    constexpr int STAGE = (2 + NB) * WB_BOX_BYTES;      // [x box of warpgroup 0][x box of warpgroup 1][NB dy boxes]
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *ring = align1024(smem_dyn);
    const int NST = p.stages;
    WideCtl &S = *reinterpret_cast<WideCtl *>(ring + (size_t)NST * STAGE);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int st = p.stride, per_img = p.n_pb * p.n_qb;

    if (threadIdx.x == 0) {
        for (int i = 0; i < NST; ++i) { bar_init(&S.full[i], 1); bar_init(&S.empty[i], WB_CONSUMER_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == WB_CONSUMER_WARPS) {
        // ===== TMA producer: per pixel block the x boxes of the unit's row blocks and the dy boxes of every filter group =====
        if (lane == 0) {
            int it = 0;
            for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
                const int split = u / p.pairs, pair = u % p.pairs;
                const int nx = 2 * pair + 1 < p.rows ? 2 : 1;
                for (int b = split_begin(p, split), b1 = split_begin(p, split + 1); b < b1; ++b, ++it) {
                    const int stage = it % NST;
                    bar_wait_relaxed(&S.empty[stage], ((unsigned)(it / NST) & 1u) ^ 1u, 32);
                    unsigned char *sp = ring + (size_t)stage * STAGE;
                    const int n = b / per_img, rem = b % per_img;
                    const int p0 = (rem / p.n_qb) * p.Pt, q0 = (rem % p.n_qb) * p.Qt;
                    bar_expect_tx(&S.full[stage], (unsigned)((nx + NB) * WB_BOX_BYTES));
                    for (int w = 0; w < nx; ++w) {
                        const int rb = 2 * pair + w, t = rb / p.nch, ch = rb % p.nch, r = t / p.S, s = t % p.S;
                        tma_load_4d(sp + w * WB_BOX_BYTES, &m.x[p.taps.rph[r] * st + p.taps.sph[s]], ch * WB_KC, q0 + p.taps.soff[s],
                                    p0 + p.taps.roff[r], n, &S.full[stage]);
                    }
                    for (int g = 0; g < NB; ++g)
                        tma_load_4d(sp + (2 + g) * WB_BOX_BYTES, &m.dy, g * 64, q0, p0, n, &S.full[stage]);
                }
            }
        }
        return;
    }

    // ===== consumer warpgroups: D[64 channels of one (tap, chunk)][N filters] += x^T[64 x 16 pixels] * dy[16 pixels x N] =====
    const int wg = warp >> 2, wq = warp & 3;
    const int RS = p.R * p.S;
    int it = 0;
    for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
        const int split = u / p.pairs, pair = u % p.pairs;
        const int rb = 2 * pair + wg;
        const bool live = rb < p.rows;                   // an odd number of row blocks leaves warpgroup 1 one idle unit
        const int b0 = split_begin(p, split), b1 = split_begin(p, split + 1);
        float acc[N / 2];
        for (int b = b0; b < b1; ++b, ++it) {
            const int stage = it % NST;
            bar_wait(&S.full[stage], (unsigned)(it / NST) & 1u);
            if (live) {
                const uint32_t sa = s_u32(ring + (size_t)stage * STAGE);
                const uint32_t a0 = sa + (uint32_t)(wg * WB_BOX_BYTES), d0 = sa + 2u * WB_BOX_BYTES;
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < 8; ++ks)            // 16 pixels = 16 rows of 128 bytes per instruction
                    wgmma_bf16<1, 1>(acc, gmma_desc_mn_sw128(a0 + ks * 2048, WB_BOX_BYTES), gmma_desc_mn_sw128(d0 + ks * 2048, WB_BOX_BYTES),
                                     (b != b0 || ks != 0) ? 1u : 0u);
                wg_commit();
            }
            if (b > b0) {                                 // the previous block's MMAs have retired: its stage is free
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
            const int t = rb / p.nch, c0 = (rb % p.nch) * WB_KC;
            float *dst = p.slots + (size_t)split * p.K * RS * p.C;
#pragma unroll
            for (int i = 0; i < N / 2; ++i) {
                const int c = c0 + wg_row(i, wq, lane), k = wg_col(i, lane);
                if (c < p.C && k < p.K) dst[((size_t)k * RS + t) * p.C + c] = acc[i];
            }
        }
    }
}

// ================================================= input gradient =======================================================
struct WideDgradParams {
    int Pt, Qt, K, nkc, G, ngroups, stride, S, stages;
    int tile0[17];                   // first tile of phase a * st + b; tile0[st * st] = all tiles
    int n_ub[16], n_vb[16];          // pixel blocks down / along the phase's grid
    int Ri[16], Sj[16];              // taps of the phase in each direction
    int rho_h[4], off_h[4];          // row phase a: taps r = rho_h[a] + tstep_h*i, dy row u - dystep_h*i + off_h[a]
    int rho_w[4], off_w[4];          // column phase b: the same with pad_w and dil_w
    int tstep_h, dystep_h;           // st/g and dil_h/g, g = gcd(dil_h, st): st and 1 at dilation 1
    int tstep_w, dystep_w;
};

// what the transposed convolution's epilogue (EPI) adds: bias [C] or NULL, the activation and the channel count C
struct WideDgradEpiParams : WideDgradParams {
    const float *bias;
    int act, C;
};

static_assert(sizeof(WideDgradEpiParams) + 18 * sizeof(CUtensorMap) <= 4096, "the input gradient's parameters exceed 4 KB");

template <bool EPI>
using DgradParamsOf = typename std::conditional<EPI, WideDgradEpiParams, WideDgradParams>::type;

struct WideDgradMaps {
    CUtensorMap dx[16];              // phase (a, b) of dx at index a * st + b: {C, ceil((W-b)/st), ceil((H-a)/st), N}
    CUtensorMap dy;                  // {K, Q, P, N}, box {64, Qt, Pt, 1}
    CUtensorMap f;                   // bf16 [R*S][C][K], box {64, N, 1}
};

struct DgradTile { int ph, n, u0, v0, g; };

__device__ __forceinline__ DgradTile dgrad_tile(const WideDgradParams &p, int tile) {
    DgradTile d;
    d.ph = 0;
    while (tile >= p.tile0[d.ph + 1]) ++d.ph;
    int rem = tile - p.tile0[d.ph];
    d.g = rem % p.ngroups;
    rem /= p.ngroups;
    const int per_img = p.n_ub[d.ph] * p.n_vb[d.ph], blk = rem % per_img;
    d.n = rem / per_img;
    d.u0 = (blk / p.n_vb[d.ph]) * p.Pt;
    d.v0 = (blk % p.n_vb[d.ph]) * p.Qt;
    return d;
}

// EPI false: the input gradient, the accumulator rounded to bf16.  EPI true: the forward of a transposed convolution, whose output
// is this input gradient, with v = accumulator + bias[c] (the accumulator itself without a bias) and the activation p.act applied in fp32 before the
// rounding, as the forward epilogues do (PCNN_ACT_*).
template <int N, bool EPI = false>   // N: channels per tile, rounded up to 16
__global__ void __launch_bounds__(WB_THREADS, 1)
k_conv_wide_dgrad(const __grid_constant__ WideDgradMaps m, const DgradParamsOf<EPI> p) {
    constexpr int NSUB = (N + 63) / 64;
    constexpr int B_BYTES = N * WB_KC * 2;
    constexpr int A_BYTES = WB_BOX_BYTES;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *stg = align1024(smem_dyn);
    unsigned char *ring = stg + 2 * NSUB * WB_STG_BYTES;
    const int NST = p.stages;
    WideCtl &S = *reinterpret_cast<WideCtl *>(ring + (size_t)NST * (A_BYTES + B_BYTES));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int st = p.stride, tiles = p.tile0[st * st];

    if (threadIdx.x == 0) {
        for (int i = 0; i < NST; ++i) { bar_init(&S.full[i], 1); bar_init(&S.empty[i], WB_CONSUMER_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == WB_CONSUMER_WARPS) {
        // ===== TMA producer: per tile and step one box of dy (shifted by the tap) and one box of filters =====
        if (lane == 0) {
            int it = 0;
            for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
                const DgradTile d = dgrad_tile(p, tile);
                const int a = d.ph / st, b = d.ph % st;
                for (int i = 0; i < p.Ri[d.ph]; ++i)
                    for (int j = 0; j < p.Sj[d.ph]; ++j) {
                        const int t = (p.rho_h[a] + p.tstep_h * i) * p.S + p.rho_w[b] + p.tstep_w * j;
                        const int bv = d.v0 - p.dystep_w * j + p.off_w[b], bu = d.u0 - p.dystep_h * i + p.off_h[a];
                        for (int kc = 0; kc < p.nkc; ++kc, ++it) {
                            const int stage = it % NST;
                            bar_wait_relaxed(&S.empty[stage], ((unsigned)(it / NST) & 1u) ^ 1u, 32);
                            unsigned char *sa = ring + (size_t)stage * (A_BYTES + B_BYTES);
                            bar_expect_tx(&S.full[stage], (unsigned)(A_BYTES + B_BYTES));
                            tma_load_4d(sa, &m.dy, kc * WB_KC, bv, bu, d.n, &S.full[stage]);
                            tma_load_3d(sa + A_BYTES, &m.f, kc * WB_KC, d.g * p.G, t, &S.full[stage]);
                        }
                    }
            }
        }
        return;
    }

    // ===== consumer warpgroups: MMA into registers, then bf16 -> staging -> TMA store into the tile's phase of dx =====
    const int wg = warp >> 2, wq = warp & 3;
    const int tid_wg = threadIdx.x & 127;
    unsigned char *my_stg = stg + (size_t)wg * NSUB * WB_STG_BYTES;
    const uint32_t stg_s = s_u32(my_stg);
    const int dp = p.Pt >= 2 ? wg * (p.Pt / 2) : 0, dq = p.Pt >= 2 ? 0 : wg * 64;
    int it = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const DgradTile d = dgrad_tile(p, tile);
        const int nsteps = p.Ri[d.ph] * p.Sj[d.ph] * p.nkc;
        float acc[N / 2];
        if (nsteps == 0) {                                // no tap reaches this phase: there is no first MMA to clear D
#pragma unroll
            for (int i = 0; i < N / 2; ++i) acc[i] = 0.0f;
        }
        for (int step = 0; step < nsteps; ++step, ++it) {
            const int stage = it % NST;
            bar_wait(&S.full[stage], (unsigned)(it / NST) & 1u);
            const uint32_t a0 = s_u32(ring + (size_t)stage * (A_BYTES + B_BYTES)) + (uint32_t)(wg * 64 * WB_KC * 2);
            const uint32_t b0 = s_u32(ring + (size_t)stage * (A_BYTES + B_BYTES) + A_BYTES);
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < WB_KC / 16; ++ks)
                wgmma_bf16<0, 0>(acc, gmma_desc_k_sw128(a0 + ks * 32), gmma_desc_k_sw128(b0 + ks * 32), (step | ks) != 0 ? 1u : 0u);
            wg_commit();
            if (step > 0) {
                wg_wait<1>();
                __syncwarp();
                if (lane == 0) bar_arrive(&S.empty[(it - 1) % NST]);
            }
        }
        if (nsteps > 0) {
            wg_wait<0>();
            wg_hold(acc);
            __syncwarp();
            if (lane == 0) bar_arrive(&S.empty[(it - 1) % NST]);
        }

        if (tid_wg == 0) bulk_wait_read0();               // the previous tile's stores have read the staging tile
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = wg_row(2 * h, wq, lane);
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
                if constexpr (EPI) {
                    const int c = d.g * p.G + wg_col(4 * j, lane);
                    if (p.bias) {
                        f0 = __fadd_rn(f0, c < p.C ? __ldg(p.bias + c) : 0.0f);
                        f1 = __fadd_rn(f1, c + 1 < p.C ? __ldg(p.bias + c + 1) : 0.0f);
                    }
                    if (p.act == PCNN_ACT_SIGMOID) { f0 = apply_act<PCNN_ACT_SIGMOID>(f0); f1 = apply_act<PCNN_ACT_SIGMOID>(f1); }
                    else if (p.act == PCNN_ACT_RELU) { f0 = apply_act<PCNN_ACT_RELU>(f0); f1 = apply_act<PCNN_ACT_RELU>(f1); }
                }
                __nv_bfloat162 v = __floats2bfloat162_rn(f0, f1);
                const uint32_t addr = stg_s + (uint32_t)((j / 8) * WB_STG_BYTES + row * 128 + (((j % 8) ^ (row & 7)) << 4) + (lane & 3) * 4);
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(*reinterpret_cast<uint32_t *>(&v)) : "memory");
            }
        }
        fence_proxy_async_smem();
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
        if (tid_wg == 0) {
#pragma unroll
            for (int sub = 0; sub < NSUB; ++sub)
                tma_store_4d(&m.dx[d.ph], my_stg + sub * WB_STG_BYTES, d.g * p.G + sub * 64, d.v0 + dq, d.u0 + dp, d.n);
            bulk_commit();
        }
    }
    if (tid_wg == 0) bulk_wait0();
}

// filters fp32 KRSC -> bf16 [R*S][C][K] (the K-major B operand of the input gradient), round to nearest even
__global__ void __launch_bounds__(256) k_wide_filters_tck(const float *__restrict__ f, __nv_bfloat16 *__restrict__ out, int K, int RS, int C) {
    const long total = (long)K * RS * C;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int k = (int)(i % K);
        const long tc = i / K;
        const int c = (int)(tc % C), t = (int)(tc / C);
        out[i] = __float2bfloat16_rn(f[((long)k * RS + t) * C + c]);
    }
}

// ================================================= host: tiling ==========================================================
size_t wgrad_stage_bytes(int n64) { return (size_t)(2 + n64 / 64) * WB_BOX_BYTES; }
size_t dgrad_staging_bytes(int n) { return 2 * (size_t)((n + 63) / 64) * WB_STG_BYTES; }
size_t dgrad_stage_bytes(int n) { return (size_t)WB_BOX_BYTES + (size_t)n * WB_KC * 2; }

struct WideBwdPlan {
    ConvWideShape sh;                 // the forward's tiling (its pixel block is the weight gradient's)
    WideWgradParams w;
    int wn;                           // weight-gradient accumulator columns (K rounded up to 64)
    WideDgradParams d;
    int dn, d_tiles;                  // input-gradient accumulator columns, tiles
};

// the taps of dx's row phase a (see the head of this file): their count, the first tap *rho and the dy offset *off
int dgrad_phase_taps(int a, int pad, int dil, int st, int R, int *rho, int *off) {
    const int g = std::gcd(dil, st), v = a + pad, tstep = st / g;
    *rho = 0;
    *off = 0;
    if (v % g != 0) return 0;
    int r = 0;
    while ((r * dil - v) % st != 0) ++r;               // r < st/g
    *rho = r;
    *off = (v - r * dil) / st;
    return r < R ? (R - r + tstep - 1) / tstep : 0;
}

int wide_bwd_plan(const char *fn, int N, int H, int W, int C, int K, int R, int S, int st, int pad_h, int pad_w, int dil_h, int dil_w,
                  int row_pitch, int image_rows, WideBwdPlan *pl) {
    memset(pl, 0, sizeof(*pl));
    int rc = conv_wide_shape(fn, N, H, W, C, K, R, S, st, pad_h, pad_w, dil_h, dil_w, row_pitch, image_rows, &pl->sh);
    if (rc) return rc;
    const ConvWideShape &sh = pl->sh;
    WideWgradParams &w = pl->w;
    w.Pt = sh.Pt; w.Qt = sh.Qt; w.n_pb = sh.n_pb; w.n_qb = sh.n_qb;
    w.R = R; w.S = S; w.stride = st; w.nch = sh.nch; w.C = C; w.K = K;
    w.taps = sh.taps;
    w.rows = R * S * sh.nch;
    w.pairs = (w.rows + 1) / 2;
    w.blocks = sh.tiles;
    w.splits = w.blocks / WB_BLOCKS_PER_SPLIT > 1 ? w.blocks / WB_BLOCKS_PER_SPLIT : 1;
    PCNN_REQUIRE((long long)w.pairs * w.splits < (1LL << 31), PCNN_ERR_ARG, "%s: work units exceed the int range", fn);
    w.units = w.pairs * w.splits;
    pl->wn = (K + 63) / 64 * 64;
    int ns = (int)(((size_t)WB_SMEM_BUDGET - sizeof(WideCtl) - 1024) / wgrad_stage_bytes(pl->wn));
    w.stages = ns > WB_MAX_STAGES ? WB_MAX_STAGES : ns;

    WideDgradParams &d = pl->d;
    d.K = K; d.nkc = (K + WB_KC - 1) / WB_KC; d.stride = st; d.S = S;
    d.ngroups = (C + WB_MAX_GROUP - 1) / WB_MAX_GROUP;
    // one group: all C channels (MMA width C rounded up to 16); several: equal widths rounded up to 64, so that the 64-channel
    // staging sub-tiles of one group never reach into the next
    d.G = d.ngroups == 1 ? C : ((C + d.ngroups - 1) / d.ngroups + 63) / 64 * 64;
    pl->dn = (d.G + 15) / 16 * 16;
    conv_wide_pixel_block((H + st - 1) / st, (W + st - 1) / st, &d.Pt, &d.Qt);    // phase (0, 0) has the largest grid
    d.tstep_h = st / std::gcd(dil_h, st); d.dystep_h = dil_h / std::gcd(dil_h, st);
    d.tstep_w = st / std::gcd(dil_w, st); d.dystep_w = dil_w / std::gcd(dil_w, st);
    int taps_h[4], taps_w[4];
    for (int a = 0; a < st; ++a) {
        taps_h[a] = dgrad_phase_taps(a, pad_h, dil_h, st, R, &d.rho_h[a], &d.off_h[a]);
        taps_w[a] = dgrad_phase_taps(a, pad_w, dil_w, st, S, &d.rho_w[a], &d.off_w[a]);
    }
    long long tiles = 0;
    for (int a = 0; a < st; ++a)
        for (int b = 0; b < st; ++b) {
            const int ph = a * st + b, U = (H - a + st - 1) / st, V = (W - b + st - 1) / st;
            d.tile0[ph] = (int)tiles;
            d.n_ub[ph] = U > 0 ? (U + d.Pt - 1) / d.Pt : 0;
            d.n_vb[ph] = V > 0 ? (V + d.Qt - 1) / d.Qt : 0;
            d.Ri[ph] = taps_h[a];
            d.Sj[ph] = taps_w[b];
            tiles += (long long)N * d.n_ub[ph] * d.n_vb[ph] * d.ngroups;
            PCNN_REQUIRE(tiles < (1LL << 31), PCNN_ERR_ARG, "%s: %lld input-gradient tiles exceed the int range", fn, tiles);
        }
    d.tile0[st * st] = (int)tiles;
    pl->d_tiles = (int)tiles;
    ns = (int)(((size_t)WB_SMEM_BUDGET - dgrad_staging_bytes(pl->dn) - sizeof(WideCtl) - 1024) / dgrad_stage_bytes(pl->dn));
    d.stages = ns > WB_MAX_STAGES ? WB_MAX_STAGES : ns;
    return PCNN_OK;
}

int dense_dy_map(CUtensorMap *map, const void *dy, int N, int P, int Q, int K, int Pt, int Qt) {
    const uint64_t dims[4] = {(uint64_t)K, (uint64_t)Q, (uint64_t)P, (uint64_t)N};
    const uint64_t str[3] = {(uint64_t)K * 2, (uint64_t)Q * K * 2, (uint64_t)P * Q * K * 2};
    const uint32_t box[4] = {WB_KC, (uint32_t)Qt, (uint32_t)Pt, 1};
    return make_map_bf16(map, const_cast<void *>(dy), 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

typedef void (*wgrad_fn)(const WideWgradMaps, const WideWgradParams);
const void *wgrad_variant(int n64) {
    static const wgrad_fn table[4] = {k_conv_wide_wgrad<64>, k_conv_wide_wgrad<128>, k_conv_wide_wgrad<192>, k_conv_wide_wgrad<256>};
    return reinterpret_cast<const void *>(table[n64 / 64 - 1]);
}
#define PCNN_DGRAD_ROW(N) \
    {reinterpret_cast<const void *>(k_conv_wide_dgrad<N, false>), reinterpret_cast<const void *>(k_conv_wide_dgrad<N, true>)}
const void *dgrad_variant(int n16, bool epi = false) {
    static const void *const table[16][2] = {
        PCNN_DGRAD_ROW(16),  PCNN_DGRAD_ROW(32),  PCNN_DGRAD_ROW(48),  PCNN_DGRAD_ROW(64),  PCNN_DGRAD_ROW(80),  PCNN_DGRAD_ROW(96),
        PCNN_DGRAD_ROW(112), PCNN_DGRAD_ROW(128), PCNN_DGRAD_ROW(144), PCNN_DGRAD_ROW(160), PCNN_DGRAD_ROW(176), PCNN_DGRAD_ROW(192),
        PCNN_DGRAD_ROW(208), PCNN_DGRAD_ROW(224), PCNN_DGRAD_ROW(240), PCNN_DGRAD_ROW(256)};
    return table[n16 / 16 - 1][epi ? 1 : 0];
}
#undef PCNN_DGRAD_ROW

int configure(pcnn_ctx *ctx) {
    static bool configured[64] = {};        // function attributes are per device
    if (!configured[ctx->device & 63]) {
        for (int v = 1; v <= 4; ++v)
            PCNN_CUDA(cudaFuncSetAttribute(wgrad_variant(64 * v), cudaFuncAttributeMaxDynamicSharedMemorySize, WB_SMEM_BUDGET + 2048));
        for (int v = 1; v <= 16; ++v)
            for (int epi = 0; epi < 2; ++epi)
                PCNN_CUDA(cudaFuncSetAttribute(dgrad_variant(16 * v, epi != 0), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               WB_SMEM_BUDGET + 2048));
        configured[ctx->device & 63] = true;
    }
    return PCNN_OK;
}

}  // namespace

// The three passes below are each entry point's body, with its name for the messages; the unpadded entry points run them at
// padding (0, 0), the unpadded and padded ones at dilation (1, 1).
static int wide_bwd_info(const char *fn, int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w, int dil_h,
                         int dil_w, int row_pitch, int image_rows, int *out10) {
    PCNN_REQUIRE(out10, PCNN_ERR_ARG, "%s: NULL argument", fn);
    WideBwdPlan pl;
    int rc = wide_bwd_plan(fn, N, H, W, C, K, R, S, stride, pad_h, pad_w, dil_h, dil_w, row_pitch, image_rows, &pl);
    if (rc) return rc;
    out10[0] = pl.w.rows; out10[1] = pl.w.splits; out10[2] = pl.w.blocks / pl.w.splits; out10[3] = pl.w.stages; out10[4] = pl.w.units;
    out10[5] = pl.d.Pt; out10[6] = pl.d.Qt; out10[7] = pl.d.ngroups; out10[8] = pl.d.stages; out10[9] = pl.d_tiles;
    return PCNN_OK;
}

static int wide_wgrad(const char *fn, pcnn_ctx *ctx, const void *x_bf16, const void *dy_bf16, float *dw_f32, int N, int H, int W, int C,
                      int K, int R, int S, int stride, int pad_h, int pad_w, int dil_h, int dil_w, int row_pitch, int image_rows) {
    PCNN_REQUIRE(ctx && x_bf16 && dy_bf16 && dw_f32, PCNN_ERR_ARG, "%s: NULL argument", fn);
    WideBwdPlan pl;
    int rc = wide_bwd_plan(fn, N, H, W, C, K, R, S, stride, pad_h, pad_w, dil_h, dil_w, row_pitch, image_rows, &pl);
    if (rc) return rc;
    PCNN_REQUIRE(((uintptr_t)x_bf16 & 15) == 0 && ((uintptr_t)dy_bf16 & 15) == 0, PCNN_ERR_ARG,
                 "%s: x and dy must be 16-byte aligned (TMA)", fn);
    pcnn_device_guard g(ctx->device);
    if ((rc = configure(ctx))) return rc;
    WideWgradParams p = pl.w;
    const int nout = K * R * S * C;
    if ((rc = pcnn_scratch(ctx, (size_t)p.splits * nout * sizeof(float), (void **)&p.slots))) return rc;
    WideWgradMaps m;
    memset(&m, 0, sizeof(m));
    if ((rc = conv_wide_x_maps(m.x, x_bf16, N, H, W, C, R, S, stride, p.taps, row_pitch, image_rows > 0 ? image_rows : H, p.Pt, p.Qt)))
        return rc;
    if ((rc = dense_dy_map(&m.dy, dy_bf16, N, pl.sh.P, pl.sh.Q, K, p.Pt, p.Qt))) return rc;
    const int grid = p.units < ctx->sm_count ? p.units : ctx->sm_count;
    void *args[] = {&m, &p};
    PCNN_CUDA(cudaLaunchKernel(wgrad_variant(pl.wn), dim3((unsigned)grid), dim3(WB_THREADS), args,
                               (size_t)p.stages * wgrad_stage_bytes(pl.wn) + sizeof(WideCtl) + 1024, ctx->stream));
    PCNN_CHECK_LAUNCH(ctx);
    return pcnn_conv_wgrad_reduce_slots(ctx, p.slots, dw_f32, p.splits, nout);
}

// epi: the transposed convolution's forward (bias may be NULL, act PCNN_ACT_*); otherwise bias and act are unused
static int wide_dgrad(const char *fn, pcnn_ctx *ctx, const void *dy_bf16, const float *filt_f32_dev, void *dx_bf16, int N, int H, int W,
                      int C, int K, int R, int S, int stride, int pad_h, int pad_w, int dil_h, int dil_w, int row_pitch, int image_rows,
                      bool epi = false, const float *bias = nullptr, int act = PCNN_ACT_NONE) {
    PCNN_REQUIRE(ctx && dy_bf16 && filt_f32_dev && dx_bf16, PCNN_ERR_ARG, "%s: NULL argument", fn);
    WideBwdPlan pl;
    int rc = wide_bwd_plan(fn, N, H, W, C, K, R, S, stride, pad_h, pad_w, dil_h, dil_w, row_pitch, image_rows, &pl);
    if (rc) return rc;
    PCNN_REQUIRE(((uintptr_t)dy_bf16 & 15) == 0 && ((uintptr_t)dx_bf16 & 15) == 0, PCNN_ERR_ARG,
                 "%s: dy and dx must be 16-byte aligned (TMA)", fn);
    pcnn_device_guard g(ctx->device);
    if ((rc = configure(ctx))) return rc;
    if (image_rows <= 0) image_rows = H;
    const int st = stride, RS = R * S;
    __nv_bfloat16 *ftck = nullptr;
    if ((rc = pcnn_scratch(ctx, (size_t)K * RS * C * 2, (void **)&ftck))) return rc;
    {
        const long total = (long)K * RS * C;
        long blocks = (total + 255) / 256;
        if (blocks > (long)ctx->sm_count * 16) blocks = (long)ctx->sm_count * 16;
        k_wide_filters_tck<<<(int)blocks, 256, 0, ctx->stream>>>(filt_f32_dev, ftck, K, RS, C);
        PCNN_CHECK_LAUNCH(ctx);
    }
    const WideDgradParams &p = pl.d;
    WideDgradMaps m;
    memset(&m, 0, sizeof(m));
    for (int a = 0; a < st; ++a)
        for (int b = 0; b < st; ++b) {
            const int ph = a * st + b;
            if (p.n_ub[ph] == 0 || p.n_vb[ph] == 0) continue;           // H or W < stride: this phase has no pixels
            const uint64_t dims[4] = {(uint64_t)C, (uint64_t)((W - b + st - 1) / st), (uint64_t)((H - a + st - 1) / st), (uint64_t)N};
            const uint64_t str[3] = {(uint64_t)st * C * 2, (uint64_t)st * row_pitch * 2, (uint64_t)image_rows * row_pitch * 2};
            const uint32_t box[4] = {64, (uint32_t)(p.Pt >= 2 ? p.Qt : 64), (uint32_t)(p.Pt >= 2 ? p.Pt / 2 : 1), 1};
            void *base = static_cast<char *>(dx_bf16) + ((size_t)a * row_pitch + (size_t)b * C) * 2;
            if ((rc = make_map_bf16(&m.dx[ph], base, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE)))
                return rc;
        }
    if ((rc = dense_dy_map(&m.dy, dy_bf16, N, pl.sh.P, pl.sh.Q, K, p.Pt, p.Qt))) return rc;
    {
        const uint64_t dims[3] = {(uint64_t)K, (uint64_t)C, (uint64_t)RS};
        const uint64_t str[2] = {(uint64_t)K * 2, (uint64_t)C * K * 2};
        const uint32_t box[3] = {WB_KC, (uint32_t)pl.dn, 1};
        if ((rc = make_map_bf16(&m.f, ftck, 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return rc;
    }
    WideDgradParams pp = p;
    WideDgradEpiParams pe;
    static_cast<WideDgradParams &>(pe) = p;
    pe.bias = bias;
    pe.act = act;
    pe.C = C;
    const int grid = pl.d_tiles < ctx->sm_count ? pl.d_tiles : ctx->sm_count;
    void *args[] = {&m, epi ? static_cast<void *>(&pe) : static_cast<void *>(&pp)};
    PCNN_CUDA(cudaLaunchKernel(dgrad_variant(pl.dn, epi), dim3((unsigned)grid), dim3(WB_THREADS), args,
                               dgrad_staging_bytes(pl.dn) + (size_t)pp.stages * dgrad_stage_bytes(pl.dn) + sizeof(WideCtl) + 1024, ctx->stream));
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_conv_wide_bwd_info(int N, int H, int W, int C, int K, int R, int S, int stride, int row_pitch, int image_rows,
                                       int *out10) {
    return wide_bwd_info("pcnn_conv_wide_bwd_info", N, H, W, C, K, R, S, stride, 0, 0, 1, 1, row_pitch, image_rows, out10);
}

extern "C" int pcnn_conv_wide_bwd_info_padded(int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w,
                                              int row_pitch, int image_rows, int *out10) {
    return wide_bwd_info("pcnn_conv_wide_bwd_info_padded", N, H, W, C, K, R, S, stride, pad_h, pad_w, 1, 1, row_pitch, image_rows, out10);
}

extern "C" int pcnn_conv_wide_bwd_info_dilated(int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w,
                                               int dil_h, int dil_w, int row_pitch, int image_rows, int *out10) {
    return wide_bwd_info("pcnn_conv_wide_bwd_info_dilated", N, H, W, C, K, R, S, stride, pad_h, pad_w, dil_h, dil_w, row_pitch,
                         image_rows, out10);
}

extern "C" int pcnn_conv_wide_wgrad(pcnn_ctx *ctx, const void *x_bf16, const void *dy_bf16, float *dw_f32, int N, int H, int W, int C,
                                    int K, int R, int S, int stride, int row_pitch, int image_rows) {
    return wide_wgrad("pcnn_conv_wide_wgrad", ctx, x_bf16, dy_bf16, dw_f32, N, H, W, C, K, R, S, stride, 0, 0, 1, 1, row_pitch,
                      image_rows);
}

extern "C" int pcnn_conv_wide_wgrad_padded(pcnn_ctx *ctx, const void *x_bf16, const void *dy_bf16, float *dw_f32, int N, int H, int W,
                                           int C, int K, int R, int S, int stride, int pad_h, int pad_w, int row_pitch, int image_rows) {
    return wide_wgrad("pcnn_conv_wide_wgrad_padded", ctx, x_bf16, dy_bf16, dw_f32, N, H, W, C, K, R, S, stride, pad_h, pad_w, 1, 1,
                      row_pitch, image_rows);
}

extern "C" int pcnn_conv_wide_wgrad_dilated(pcnn_ctx *ctx, const void *x_bf16, const void *dy_bf16, float *dw_f32, int N, int H, int W,
                                            int C, int K, int R, int S, int stride, int pad_h, int pad_w, int dil_h, int dil_w,
                                            int row_pitch, int image_rows) {
    return wide_wgrad("pcnn_conv_wide_wgrad_dilated", ctx, x_bf16, dy_bf16, dw_f32, N, H, W, C, K, R, S, stride, pad_h, pad_w, dil_h,
                      dil_w, row_pitch, image_rows);
}

extern "C" int pcnn_conv_wide_dgrad(pcnn_ctx *ctx, const void *dy_bf16, const float *filt_f32_dev, void *dx_bf16, int N, int H, int W,
                                    int C, int K, int R, int S, int stride, int row_pitch, int image_rows) {
    return wide_dgrad("pcnn_conv_wide_dgrad", ctx, dy_bf16, filt_f32_dev, dx_bf16, N, H, W, C, K, R, S, stride, 0, 0, 1, 1, row_pitch,
                      image_rows);
}

extern "C" int pcnn_conv_wide_dgrad_padded(pcnn_ctx *ctx, const void *dy_bf16, const float *filt_f32_dev, void *dx_bf16, int N, int H,
                                           int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w, int row_pitch,
                                           int image_rows) {
    return wide_dgrad("pcnn_conv_wide_dgrad_padded", ctx, dy_bf16, filt_f32_dev, dx_bf16, N, H, W, C, K, R, S, stride, pad_h, pad_w, 1,
                      1, row_pitch, image_rows);
}

extern "C" int pcnn_conv_wide_dgrad_dilated(pcnn_ctx *ctx, const void *dy_bf16, const float *filt_f32_dev, void *dx_bf16, int N, int H,
                                            int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w, int dil_h, int dil_w,
                                            int row_pitch, int image_rows) {
    return wide_dgrad("pcnn_conv_wide_dgrad_dilated", ctx, dy_bf16, filt_f32_dev, dx_bf16, N, H, W, C, K, R, S, stride, pad_h, pad_w,
                      dil_h, dil_w, row_pitch, image_rows);
}

// ================================================= transposed convolution ===============================================
// conv_transpose2d(x, w, b, stride, padding, output_padding) is the input gradient of its adjoint convolution: input H_out x W_out
// x C_out, K = C_in filters f[ci][r][s][co] = w[ci][co][r][s], the same stride and padding, whose output is H x W.  The rules below
// are stated in the transposed convolution's own terms before the adjoint's shape rules (pitch, plan split) are checked.
static int conv_transpose_shape(const char *fn, int N, int H, int W, int C_in, int C_out, int R, int S, int stride, int pad_h, int pad_w,
                                int op_h, int op_w, int has_bias, int act, int *H_out, int *W_out, WideBwdPlan *pl, int row_pitch,
                                int image_rows) {
    PCNN_REQUIRE(N >= 1 && H >= 1 && W >= 1, PCNN_ERR_ARG, "%s: N = %d, H = %d, W = %d: each must be >= 1", fn, N, H, W);
    PCNN_REQUIRE(C_in >= 8 && C_in % 8 == 0 && C_in <= 256, PCNN_ERR_ARG,
                 "%s: C_in = %d: C_in %% 8 == 0 and 8 <= C_in <= 256 are required (the adjoint convolution's filters)", fn, C_in);
    PCNN_REQUIRE(C_out >= 8 && C_out % 8 == 0, PCNN_ERR_ARG, "%s: C_out = %d: C_out %% 8 == 0 and C_out >= 8 are required", fn, C_out);
    PCNN_REQUIRE(!(has_bias || act != PCNN_ACT_NONE) || C_out <= 256, PCNN_ERR_ARG,
                 "%s: C_out = %d with a bias or an activation: C_out <= 256 is required (pcnn_conv_bias_act_bwd)", fn, C_out);
    PCNN_REQUIRE_ACT(fn, act);
    PCNN_REQUIRE(stride >= 1 && stride <= 4, PCNN_ERR_ARG, "%s: stride %d outside 1..4", fn, stride);
    PCNN_REQUIRE(R >= 1 && R <= 7 && S >= 1 && S <= 7, PCNN_ERR_ARG, "%s: R = %d, S = %d: taps must be 1..7 in each direction", fn, R, S);
    PCNN_REQUIRE(pad_h >= 0 && pad_h < R && pad_w >= 0 && pad_w < S, PCNN_ERR_ARG,
                 "%s: padding (%d, %d) with R = %d, S = %d taps: 0 <= pad_h <= R - 1 and 0 <= pad_w <= S - 1 are required", fn, pad_h,
                 pad_w, R, S);
    PCNN_REQUIRE(op_h >= 0 && op_h < stride && op_w >= 0 && op_w < stride, PCNN_ERR_ARG,
                 "%s: output_padding (%d, %d) at stride %d: 0 <= output_padding < stride is required", fn, op_h, op_w, stride);
    const long long ho = (long long)(H - 1) * stride - 2LL * pad_h + R + op_h, wo = (long long)(W - 1) * stride - 2LL * pad_w + S + op_w;
    PCNN_REQUIRE(ho >= 1 && wo >= 1 && ho < (1 << 24) && wo < (1 << 24), PCNN_ERR_ARG,
                 "%s: output %lld x %lld: H_out = (H - 1) stride - 2 pad_h + R + output_padding_h (and W_out the same) must be 1 .. 2^24 - 1",
                 fn, ho, wo);
    PCNN_REQUIRE((pad_h == 0 || ho >= stride) && (pad_w == 0 || wo >= stride), PCNN_ERR_ARG,
                 "%s: output %lld x %lld with padding (%d, %d) at stride %d: a padded direction needs an output of at least stride "
                 "rows / pixels", fn, ho, wo, pad_h, pad_w, stride);
    *H_out = (int)ho;
    *W_out = (int)wo;
    return wide_bwd_plan(fn, N, (int)ho, (int)wo, C_out, C_in, R, S, stride, pad_h, pad_w, 1, 1,
                         row_pitch == 0 ? (int)wo * C_out : row_pitch, image_rows, pl);
}

extern "C" int pcnn_conv_transpose_info(int N, int H, int W, int C_in, int C_out, int R, int S, int stride, int pad_h, int pad_w, int op_h,
                                        int op_w, int row_pitch, int image_rows, int has_bias, int act, int *out8) {
    const char *fn = "pcnn_conv_transpose_info";
    PCNN_REQUIRE(out8, PCNN_ERR_ARG, "%s: NULL out8", fn);
    WideBwdPlan pl;
    int ho, wo;
    const int rc = conv_transpose_shape(fn, N, H, W, C_in, C_out, R, S, stride, pad_h, pad_w, op_h, op_w, has_bias, act, &ho, &wo, &pl,
                                        row_pitch, image_rows);
    if (rc) return rc;
    out8[0] = ho; out8[1] = wo;
    out8[2] = row_pitch == 0 ? wo * C_out : row_pitch; out8[3] = image_rows > 0 ? image_rows : ho;
    out8[4] = pl.d.Pt; out8[5] = pl.d.Qt; out8[6] = pl.d.ngroups; out8[7] = pl.d_tiles;
    return PCNN_OK;
}

extern "C" int pcnn_conv_transpose_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, const float *filt_f32_dev, const float *bias_f32_dev,
                                       void *y_bf16_dev, int N, int H, int W, int C_in, int C_out, int R, int S, int stride, int pad_h,
                                       int pad_w, int op_h, int op_w, int row_pitch, int image_rows, int act) {
    const char *fn = "pcnn_conv_transpose_fwd";
    PCNN_REQUIRE(ctx && x_bf16_dev && filt_f32_dev && y_bf16_dev, PCNN_ERR_ARG, "%s: NULL context, x, filters or y (only the bias may be NULL)",
                 fn);
    WideBwdPlan pl;
    int ho, wo;
    const int rc = conv_transpose_shape(fn, N, H, W, C_in, C_out, R, S, stride, pad_h, pad_w, op_h, op_w, bias_f32_dev != nullptr, act, &ho,
                                        &wo, &pl, row_pitch, image_rows);
    if (rc) return rc;
    return wide_dgrad(fn, ctx, x_bf16_dev, filt_f32_dev, y_bf16_dev, N, ho, wo, C_out, C_in, R, S, stride, pad_h, pad_w, 1, 1,
                      row_pitch == 0 ? wo * C_out : row_pitch, image_rows, true, bias_f32_dev, act);
}
