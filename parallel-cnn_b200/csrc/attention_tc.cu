// parallel-cnn_b200/csrc/attention_tc.cu -- self-attention over the pixels of each image on the Hopper tensor cores
// (pcnn_attention_bf16_fwd, pcnn_attention_bf16_bwd, pcnn_attention_info).  sm_90a.
//
// Per image n and head j, with T tokens (the pixels, NHWC order) and head size D: O = softmax(scale Q K^T) V.  q, k and v are bf16
// rows of `ld` elements, element (n, t, j, i) at (n T + t) ld + j D + i; a 4-D tensor map {D, heads, T, N} over each returns a
// box of 64 tokens of one head with zero fill past T.  Every operand tile in shared memory is 64 rows x D: D / 64 column boxes of
// 64 rows x 128 B (SWIZZLE_128B) for D >= 64, one box of 64 rows x 2D bytes (SWIZZLE_64B / _32B) for D = 32 / 16.  The same tile
// serves as a K-major operand (reduction over D) and as an MN-major B operand (reduction over its 64 rows).
//
//   * Forward (k_attn_fwd): a tile is (n, j, block of 64 NWG query rows), one warpgroup per 64 rows.  It loops over key blocks of
//     64: S = Q K^T (both K-major), the online max and sum in fp32, P rounded to bf16 in registers and O += P V with P as the
//     register A operand and V MN-major.  Keys >= T (zero-filled) get -inf before the row max.
//   * Backward: k_attn_dsum forms D = sum_i dO O per row.  k_attn_dkdv: a tile is (n, j, block of 64 NWG keys); it loops over
//     query blocks of 64 with S^T = K Q^T and dP^T = V dO^T, recomputes P^T from lse, dV += P^T dO and dK += dS^T Q.
//     k_attn_dq: a tile is (n, j, block of 64 NWG queries); it loops over key blocks with S = Q K^T and dP = dO V^T and
//     accumulates dQ += dS K.  No atomics; each tile loops in a fixed order, so the bits of one (n, j) depend on nothing else.
// Warp roles (NWG * 128 + 32 threads, persistent over tiles): NWG consumer warpgroups, then one TMA producer warp.
#include "tc_common.cuh"

#include <cuda_bf16.h>
#include <cmath>
#include <math.h>

using namespace pcnn_tc;

namespace {

constexpr int AT_ROWS = 64;               // rows of a tile per warpgroup, and of every streamed block
constexpr int AT_STAGES = 2;              // streamed blocks in flight
constexpr int AT_NWG = 2;                 // consumer warpgroups of every kernel
constexpr int AT_THREADS = AT_NWG * 128 + 32;
constexpr int AT_MAX_T = 16384;

template <int D>
struct Geo {
    static constexpr int RB = D < 64 ? 2 * D : 128;          // bytes per row of one column box
    static constexpr int NBOX = D > 64 ? D / 64 : 1;
    static constexpr int BOXC = RB / 2;                       // columns per box
    static constexpr int BOXB = AT_ROWS * RB;
    static constexpr int TILE = NBOX * BOXB;                  // one 64 x D tile
    static constexpr uint32_t LT = RB == 128 ? 1u : RB == 64 ? 2u : 3u;   // SWIZZLE_128B / _64B / _32B
};

// K-major operand (rows of D elements), K step ks of 16 elements
template <int D> __device__ __forceinline__ uint64_t desc_k(uint32_t tile, int ks) {
    using G = Geo<D>;
    return gmma_desc(tile + (uint32_t)((ks * 32 / G::RB) * G::BOXB + (ks * 32) % G::RB), 16, 8 * G::RB, G::LT);
}
// MN-major B operand (N = D along the rows, K = the tile's 64 rows), K step ks of 16 rows
template <int D> __device__ __forceinline__ uint64_t desc_mn(uint32_t tile, int ks) {
    using G = Geo<D>;
    return gmma_desc(tile + (uint32_t)(ks * 16 * G::RB), G::BOXB, 8 * G::RB, G::LT);
}

__device__ __forceinline__ float ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float lg2(float x) {
    float y;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t *>(&h);
}

struct AtCtl {
    unsigned long long full[AT_STAGES], empty[AT_STAGES], tfull, tempty;
};

struct AttnMaps {
    CUtensorMap q, k, v, dout;
};

struct AttnParams {
    int T, h, nblk, tiles;       // nblk: tiles per (n, j)
    float c2, scale;             // c2 = RN(scale log2 e)
    __nv_bfloat16 *o;            // forward: [N][T][h][D]
    float *lse;                  // forward: [N][h][T]
    const float *lse_in, *dsum;  // backward: [N][h][T]
    __nv_bfloat16 *dq, *dk, *dv; // backward, rows of ld_g
    long ldg;
};

__device__ __forceinline__ unsigned char *align1024(unsigned char *p) {
    return reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(p) + 1023) & ~(uintptr_t)1023);
}

template <int D>
__device__ __forceinline__ void load_tile(unsigned char *dst, const CUtensorMap *map, int j, int row, int n, unsigned long long *bar) {
    using G = Geo<D>;
#pragma unroll
    for (int b = 0; b < G::NBOX; ++b) tma_load_4d(dst + b * G::BOXB, map, b * G::BOXC, j, row, n, bar);
}

__device__ __forceinline__ void init_bars(AtCtl &S) {
    if (threadIdx.x == 0) {
        for (int i = 0; i < AT_STAGES; ++i) { bar_init(&S.full[i], 1); bar_init(&S.empty[i], AT_NWG * 4); }
        bar_init(&S.tfull, 1);
        bar_init(&S.tempty, AT_NWG * 4);
        fence_barrier_init();
    }
    __syncthreads();
}

// The producer of all three kernels: per tile, `per_tile` tiles of the fixed operands (a: rows of this warpgroup's block, from
// maps ta and tb), then the T / 64 streamed blocks, each a pair of tiles from maps sa and sb.
template <int D, int FIXED>
__device__ __forceinline__ void produce(unsigned char *fixed, unsigned char *ring, AtCtl &S, const CUtensorMap *ta, const CUtensorMap *tb,
                                        const CUtensorMap *sa, const CUtensorMap *sb, const AttnParams &p) {
    using G = Geo<D>;
    const int nsb = (p.T + AT_ROWS - 1) / AT_ROWS;
    int it = 0, tc = 0;
    for (int u = blockIdx.x; u < p.tiles; u += gridDim.x, ++tc) {
        const int blk = u % p.nblk, nj = u / p.nblk, j = nj % p.h, n = nj / p.h;
        bar_wait_relaxed(&S.tempty, ((unsigned)tc & 1u) ^ 1u, 32);
        bar_expect_tx(&S.tfull, (unsigned)(FIXED * AT_NWG * G::TILE));
        for (int w = 0; w < AT_NWG; ++w) {
            const int row = (blk * AT_NWG + w) * AT_ROWS;
            load_tile<D>(fixed + w * G::TILE, ta, j, row, n, &S.tfull);
            if (FIXED == 2) load_tile<D>(fixed + (AT_NWG + w) * G::TILE, tb, j, row, n, &S.tfull);
        }
        for (int b = 0; b < nsb; ++b, ++it) {
            const int stage = it % AT_STAGES;
            bar_wait_relaxed(&S.empty[stage], ((unsigned)(it / AT_STAGES) & 1u) ^ 1u, 32);
            unsigned char *st = ring + (size_t)stage * 2 * G::TILE;
            bar_expect_tx(&S.full[stage], (unsigned)(2 * G::TILE));
            load_tile<D>(st, sa, j, b * AT_ROWS, n, &S.full[stage]);
            load_tile<D>(st + G::TILE, sb, j, b * AT_ROWS, n, &S.full[stage]);
        }
    }
}

__device__ __forceinline__ void release(unsigned long long *bar, int lane) {
    __syncwarp();
    if (lane == 0) bar_arrive(bar);
}

// ================================================= forward =====================================================================
template <int D>
__global__ void __launch_bounds__(AT_THREADS, 1) k_attn_fwd(const __grid_constant__ AttnMaps m, const AttnParams p) {
    using G = Geo<D>;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *qs = align1024(smem_dyn);                 // [NWG] Q tiles
    unsigned char *ring = qs + AT_NWG * G::TILE;             // [stages][K tile, V tile]
    AtCtl &S = *reinterpret_cast<AtCtl *>(ring + AT_STAGES * 2 * G::TILE);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    init_bars(S);
    if (warp == AT_NWG * 4) {
        if (lane == 0) produce<D, 1>(qs, ring, S, &m.q, nullptr, &m.k, &m.v, p);
        return;
    }
    const int wg = warp >> 2, wq = warp & 3;
    const int nkb = (p.T + AT_ROWS - 1) / AT_ROWS;
    int it = 0, tc = 0;
    for (int u = blockIdx.x; u < p.tiles; u += gridDim.x, ++tc) {
        const int blk = u % p.nblk, nj = u / p.nblk, j = nj % p.h, n = nj / p.h;
        bar_wait(&S.tfull, (unsigned)tc & 1u);
        const uint32_t qa = s_u32(qs + wg * G::TILE);
        float o[D / 2], mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.0f, 0.0f};
#pragma unroll
        for (int i = 0; i < D / 2; ++i) o[i] = 0.0f;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
            const int stage = it % AT_STAGES;
            bar_wait(&S.full[stage], (unsigned)(it / AT_STAGES) & 1u);
            const uint32_t ka = s_u32(ring + (size_t)stage * 2 * G::TILE), va = ka + G::TILE;
            float s[32];
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < D / 16; ++ks) wgmma_bf16<0, 0>(s, desc_k<D>(qa, ks), desc_k<D>(ka, ks), ks > 0 ? 1u : 0u);
            wg_commit();
            wg_wait<0>();
            wg_hold(s);
            // base-2 logits u = RN(s c2); keys past T (zero-filled rows of K) are -inf before the row max
            float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                const int key = kb * AT_ROWS + wg_col(i, lane);
                s[i] = key < p.T ? __fmul_rn(s[i], p.c2) : -INFINITY;
                mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
            }
            float alpha[2], rs[2] = {0.0f, 0.0f};
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
                const float mnew = fmaxf(mrow[r], mx[r]);
                alpha[r] = ex2(__fsub_rn(mrow[r], mnew));        // the first block: ex2(-inf) = 0
                mrow[r] = mnew;
            }
            uint32_t pa[16];
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
                const int r = (i >> 1) & 1;
                pa[i / 2] = pack_bf16(ex2(__fsub_rn(s[i], mrow[r])), ex2(__fsub_rn(s[i + 1], mrow[r])));
                const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162 *>(&pa[i / 2]);
                rs[r] = __fadd_rn(__fadd_rn(rs[r], __low2float(h)), __high2float(h));
            }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                rs[r] = __fadd_rn(rs[r], __shfl_xor_sync(0xffffffffu, rs[r], 1));
                rs[r] = __fadd_rn(rs[r], __shfl_xor_sync(0xffffffffu, rs[r], 2));
                lrow[r] = __fadd_rn(__fmul_rn(lrow[r], alpha[r]), rs[r]);
            }
#pragma unroll
            for (int i = 0; i < D / 2; ++i) o[i] = __fmul_rn(o[i], alpha[(i >> 1) & 1]);
            wg_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
                wgmma_bf16_rs<1>(o, a, desc_mn<D>(va, kk), 1u);
            }
            wg_commit();
            wg_wait<0>();
            wg_hold(o);
            release(&S.empty[stage], lane);
        }
        release(&S.tempty, lane);
        const int row0 = (blk * AT_NWG + wg) * AT_ROWS;
        const float inv[2] = {__frcp_rn(lrow[0]), __frcp_rn(lrow[1])};
#pragma unroll
        for (int i = 0; i < D / 2; i += 2) {
            const int r = (i >> 1) & 1, t = row0 + wg_row(i, wq, lane);
            if (t >= p.T) continue;
            __nv_bfloat16 *dst = p.o + ((size_t)n * p.T + t) * ((size_t)p.h * D) + (size_t)j * D + wg_col(i, lane);
            *reinterpret_cast<__nv_bfloat162 *>(dst) = __floats2bfloat162_rn(__fmul_rn(o[i], inv[r]), __fmul_rn(o[i + 1], inv[r]));
        }
        if ((lane & 3) == 0) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int t = row0 + 16 * wq + (lane >> 2) + 8 * r;
                if (t < p.T) p.lse[((size_t)n * p.h + j) * p.T + t] = __fmul_rn(__fadd_rn(mrow[r], lg2(lrow[r])), 0.69314718055994531f);
            }
        }
    }
}

// ================================================= backward ====================================================================
// dsum[n][j][t] = sum over i = 0 .. D - 1 of float(dO) float(O), fp32 fma in that order
__global__ void __launch_bounds__(256) k_attn_dsum(const __nv_bfloat16 *__restrict__ o, const __nv_bfloat16 *__restrict__ dout,
                                                   float *__restrict__ dsum, long rows, int T, int h, int D) {
    for (long r = blockIdx.x * 256L + threadIdx.x; r < rows; r += (long)gridDim.x * 256) {   // r = (n T + t) h + j
        const __nv_bfloat16 *a = o + r * D, *b = dout + r * D;
        float acc = 0.0f;
        for (int i = 0; i < D; i += 2) {
            const float2 x = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(a + i));
            const float2 y = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(b + i));
            acc = __fmaf_rn(y.x, x.x, acc);
            acc = __fmaf_rn(y.y, x.y, acc);
        }
        const long nt = r / h, n = nt / T, t = nt % T;
        const int j = (int)(r % h);
        dsum[((size_t)n * h + j) * T + t] = acc;
    }
}

// P = ex2(RN(RN(s c2) - l2)) with l2 = RN(lse log2 e), 0 past T; dS = RN(P RN(dP - Dsum)); both returned packed as bf16 pairs
__device__ __forceinline__ void p_ds(float s0, float s1, float dp0, float dp1, float l0, float l1, float d0, float d1, bool v0, bool v1,
                                     float c2, uint32_t &pp, uint32_t &dd) {
    const float p0 = v0 ? ex2(__fsub_rn(__fmul_rn(s0, c2), l0)) : 0.0f;
    const float p1 = v1 ? ex2(__fsub_rn(__fmul_rn(s1, c2), l1)) : 0.0f;
    pp = pack_bf16(p0, p1);
    dd = pack_bf16(__fmul_rn(p0, __fsub_rn(dp0, d0)), __fmul_rn(p1, __fsub_rn(dp1, d1)));
}

template <int D>
__device__ __forceinline__ void store_rows(__nv_bfloat16 *base, long ldg, const float (&acc)[D / 2], float mul, int n, int T, int j,
                                           int row0, int wq, int lane) {
#pragma unroll
    for (int i = 0; i < D / 2; i += 2) {
        const int t = row0 + wg_row(i, wq, lane);
        if (t >= T) continue;
        __nv_bfloat16 *dst = base + ((size_t)n * T + t) * ldg + (size_t)j * D + wg_col(i, lane);
        *reinterpret_cast<__nv_bfloat162 *>(dst) = __floats2bfloat162_rn(__fmul_rn(acc[i], mul), __fmul_rn(acc[i + 1], mul));
    }
}

template <int D>
__global__ void __launch_bounds__(AT_THREADS, 1) k_attn_dkdv(const __grid_constant__ AttnMaps m, const AttnParams p) {
    using G = Geo<D>;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *fixed = align1024(smem_dyn);              // [NWG] K tiles, [NWG] V tiles
    unsigned char *ring = fixed + 2 * AT_NWG * G::TILE;      // [stages][Q tile, dO tile]
    AtCtl &S = *reinterpret_cast<AtCtl *>(ring + AT_STAGES * 2 * G::TILE);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    init_bars(S);
    if (warp == AT_NWG * 4) {
        if (lane == 0) produce<D, 2>(fixed, ring, S, &m.k, &m.v, &m.q, &m.dout, p);
        return;
    }
    const int wg = warp >> 2, wq = warp & 3;
    const int nqb = (p.T + AT_ROWS - 1) / AT_ROWS;
    int it = 0, tc = 0;
    for (int u = blockIdx.x; u < p.tiles; u += gridDim.x, ++tc) {
        const int blk = u % p.nblk, nj = u / p.nblk, j = nj % p.h, n = nj / p.h;
        const float *L = p.lse_in + ((size_t)n * p.h + j) * p.T, *Ds = p.dsum + ((size_t)n * p.h + j) * p.T;
        bar_wait(&S.tfull, (unsigned)tc & 1u);
        const uint32_t ka = s_u32(fixed + wg * G::TILE), va = s_u32(fixed + (AT_NWG + wg) * G::TILE);
        float dk[D / 2], dv[D / 2];
#pragma unroll
        for (int i = 0; i < D / 2; ++i) dk[i] = dv[i] = 0.0f;
        for (int qb = 0; qb < nqb; ++qb, ++it) {
            const int stage = it % AT_STAGES;
            bar_wait(&S.full[stage], (unsigned)(it / AT_STAGES) & 1u);
            const uint32_t qa = s_u32(ring + (size_t)stage * 2 * G::TILE), da = qa + G::TILE;
            float st[32], dpt[32];
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < D / 16; ++ks) wgmma_bf16<0, 0>(st, desc_k<D>(ka, ks), desc_k<D>(qa, ks), ks > 0 ? 1u : 0u);
#pragma unroll
            for (int ks = 0; ks < D / 16; ++ks) wgmma_bf16<0, 0>(dpt, desc_k<D>(va, ks), desc_k<D>(da, ks), ks > 0 ? 1u : 0u);
            wg_commit();
            wg_wait<0>();
            wg_hold(st);
            wg_hold(dpt);
            uint32_t pa[16], sa[16];
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
                // the columns are queries q and q + 1, with their RN(lse log2 e) and Dsum
                const int q = qb * AT_ROWS + wg_col(i, lane);
                const bool v0 = q < p.T, v1 = q + 1 < p.T;
                const float l0 = v0 ? __fmul_rn(__ldg(L + q), 1.4426950408889634f) : 0.0f, l1 = v1 ? __fmul_rn(__ldg(L + q + 1), 1.4426950408889634f) : 0.0f;
                p_ds(st[i], st[i + 1], dpt[i], dpt[i + 1], l0, l1, v0 ? __ldg(Ds + q) : 0.0f, v1 ? __ldg(Ds + q + 1) : 0.0f, v0, v1, p.c2,
                     pa[i / 2], sa[i / 2]);
            }
            wg_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
                wgmma_bf16_rs<1>(dv, a, desc_mn<D>(da, kk), 1u);
            }
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t a[4] = {sa[4 * kk], sa[4 * kk + 1], sa[4 * kk + 2], sa[4 * kk + 3]};
                wgmma_bf16_rs<1>(dk, a, desc_mn<D>(qa, kk), 1u);
            }
            wg_commit();
            wg_wait<0>();
            wg_hold(dv);
            wg_hold(dk);
            release(&S.empty[stage], lane);
        }
        release(&S.tempty, lane);
        const int row0 = (blk * AT_NWG + wg) * AT_ROWS;
        store_rows<D>(p.dk, p.ldg, dk, p.scale, n, p.T, j, row0, wq, lane);
        store_rows<D>(p.dv, p.ldg, dv, 1.0f, n, p.T, j, row0, wq, lane);
    }
}

template <int D>
__global__ void __launch_bounds__(AT_THREADS, 1) k_attn_dq(const __grid_constant__ AttnMaps m, const AttnParams p) {
    using G = Geo<D>;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *fixed = align1024(smem_dyn);              // [NWG] Q tiles, [NWG] dO tiles
    unsigned char *ring = fixed + 2 * AT_NWG * G::TILE;      // [stages][K tile, V tile]
    AtCtl &S = *reinterpret_cast<AtCtl *>(ring + AT_STAGES * 2 * G::TILE);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    init_bars(S);
    if (warp == AT_NWG * 4) {
        if (lane == 0) produce<D, 2>(fixed, ring, S, &m.q, &m.dout, &m.k, &m.v, p);
        return;
    }
    const int wg = warp >> 2, wq = warp & 3;
    const int nkb = (p.T + AT_ROWS - 1) / AT_ROWS;
    int it = 0, tc = 0;
    for (int u = blockIdx.x; u < p.tiles; u += gridDim.x, ++tc) {
        const int blk = u % p.nblk, nj = u / p.nblk, j = nj % p.h, n = nj / p.h;
        const int row0 = (blk * AT_NWG + wg) * AT_ROWS;
        float l2[2], dd[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int t = row0 + 16 * wq + (lane >> 2) + 8 * r;
            const size_t at = ((size_t)n * p.h + j) * p.T + t;
            l2[r] = t < p.T ? __fmul_rn(p.lse_in[at], 1.4426950408889634f) : 0.0f;
            dd[r] = t < p.T ? p.dsum[at] : 0.0f;
        }
        bar_wait(&S.tfull, (unsigned)tc & 1u);
        const uint32_t qa = s_u32(fixed + wg * G::TILE), oa = s_u32(fixed + (AT_NWG + wg) * G::TILE);
        float dq[D / 2];
#pragma unroll
        for (int i = 0; i < D / 2; ++i) dq[i] = 0.0f;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
            const int stage = it % AT_STAGES;
            bar_wait(&S.full[stage], (unsigned)(it / AT_STAGES) & 1u);
            const uint32_t ka = s_u32(ring + (size_t)stage * 2 * G::TILE), va = ka + G::TILE;
            float s[32], dp[32];
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < D / 16; ++ks) wgmma_bf16<0, 0>(s, desc_k<D>(qa, ks), desc_k<D>(ka, ks), ks > 0 ? 1u : 0u);
#pragma unroll
            for (int ks = 0; ks < D / 16; ++ks) wgmma_bf16<0, 0>(dp, desc_k<D>(oa, ks), desc_k<D>(va, ks), ks > 0 ? 1u : 0u);
            wg_commit();
            wg_wait<0>();
            wg_hold(s);
            wg_hold(dp);
            uint32_t pa[16], sa[16];
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
                const int r = (i >> 1) & 1, key = kb * AT_ROWS + wg_col(i, lane);
                p_ds(s[i], s[i + 1], dp[i], dp[i + 1], l2[r], l2[r], dd[r], dd[r], key < p.T, key + 1 < p.T, p.c2, pa[i / 2], sa[i / 2]);
            }
            wg_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t a[4] = {sa[4 * kk], sa[4 * kk + 1], sa[4 * kk + 2], sa[4 * kk + 3]};
                wgmma_bf16_rs<1>(dq, a, desc_mn<D>(ka, kk), 1u);
            }
            wg_commit();
            wg_wait<0>();
            wg_hold(dq);
            release(&S.empty[stage], lane);
        }
        release(&S.tempty, lane);
        store_rows<D>(p.dq, p.ldg, dq, p.scale, n, p.T, j, row0, wq, lane);
    }
}

}  // namespace

// ================================================= host ==========================================================================
struct AttnShape {
    int N, T, h, d, ld, ldg, nblk, tiles;
    float c2;
    size_t scratch;
};

static int smem_fwd(int d) { return AT_NWG * 64 * d * 2 + AT_STAGES * 2 * 64 * d * 2 + (int)sizeof(AtCtl) + 1024; }
static int smem_bwd(int d) { return 2 * AT_NWG * 64 * d * 2 + AT_STAGES * 2 * 64 * d * 2 + (int)sizeof(AtCtl) + 1024; }

// the domain of the three calls (the refusals name `fn`) and the partition, a function of the shape alone; ldg 0: not checked
static int attn_shape(const char *fn, int N, int T, int h, int d, int ld, int ldg, float scale, AttnShape *s) {
    PCNN_REQUIRE(d == 16 || d == 32 || d == 64 || d == 128, PCNN_ERR_ARG, "%s: head size d = %d: 16, 32, 64 or 128 is required", fn, d);
    PCNN_REQUIRE(h >= 1, PCNN_ERR_ARG, "%s: heads = %d: at least 1 is required", fn, h);
    PCNN_REQUIRE(N >= 1, PCNN_ERR_ARG, "%s: N = %d: at least one image is required", fn, N);
    PCNN_REQUIRE(T >= 1 && T <= AT_MAX_T, PCNN_ERR_ARG, "%s: T = %d tokens: 1 <= T <= %d is required", fn, T, AT_MAX_T);
    const long long hd = (long long)h * d;
    PCNN_REQUIRE(ld >= hd && ld % 8 == 0, PCNN_ERR_ARG, "%s: ld = %d: a multiple of 8 elements and >= heads * d = %lld is required", fn,
                 ld, hd);
    PCNN_REQUIRE(ldg == 0 || (ldg >= hd && ldg % 8 == 0), PCNN_ERR_ARG,
                 "%s: ld_g = %d: a multiple of 8 elements and >= heads * d = %lld is required", fn, ldg, hd);
    PCNN_REQUIRE(std::isfinite(scale) && scale > 0.0f, PCNN_ERR_ARG, "%s: scale = %g: a finite scale > 0 is required", fn, (double)scale);
    const int rows = AT_NWG * AT_ROWS;
    const long long tiles = (long long)N * h * ((T + rows - 1) / rows);
    PCNN_REQUIRE(tiles < (1LL << 31), PCNN_ERR_ARG, "%s: N * heads * ceil(T / %d) = %lld tiles: fewer than 2^31 are required", fn, rows,
                 tiles);
    s->N = N; s->T = T; s->h = h; s->d = d; s->ld = ld; s->ldg = ldg;
    s->nblk = (T + rows - 1) / rows;
    s->tiles = (int)tiles;
    s->c2 = (float)((double)scale * 1.4426950408889634);
    s->scratch = (size_t)N * h * T * sizeof(float);
    return PCNN_OK;
}

extern "C" int pcnn_attention_info(int N, int T, int heads, int d, int ld, int ld_g, float scale, long long *out8) {
    const char *fn = "pcnn_attention_info";
    PCNN_REQUIRE(out8, PCNN_ERR_ARG, "%s: NULL argument", fn);
    AttnShape s;
    int rc = attn_shape(fn, N, T, heads, d, ld, ld_g, scale, &s);
    if (rc) return rc;
    const long long v[8] = {AT_NWG * AT_ROWS, AT_ROWS, AT_STAGES, s.tiles, s.tiles, s.tiles, (long long)s.scratch, smem_bwd(d)};
    memcpy(out8, v, sizeof(v));
    return PCNN_OK;
}

typedef void (*attn_fn)(const AttnMaps, const AttnParams);
static const void *variant(int which, int d) {   // which: 0 forward, 1 dK dV, 2 dQ
    static const attn_fn t[3][4] = {{k_attn_fwd<16>, k_attn_fwd<32>, k_attn_fwd<64>, k_attn_fwd<128>},
                                    {k_attn_dkdv<16>, k_attn_dkdv<32>, k_attn_dkdv<64>, k_attn_dkdv<128>},
                                    {k_attn_dq<16>, k_attn_dq<32>, k_attn_dq<64>, k_attn_dq<128>}};
    const int i = d == 16 ? 0 : d == 32 ? 1 : d == 64 ? 2 : 3;
    return reinterpret_cast<const void *>(t[which][i]);
}

static int configure(pcnn_ctx *ctx) {
    static bool configured[64] = {};        // function attributes are per device
    if (configured[ctx->device & 63]) return PCNN_OK;
    for (int d = 16; d <= 128; d *= 2)
        for (int w = 0; w < 3; ++w)
            PCNN_CUDA(cudaFuncSetAttribute(variant(w, d), cudaFuncAttributeMaxDynamicSharedMemorySize, w ? smem_bwd(d) : smem_fwd(d)));
    configured[ctx->device & 63] = true;
    return PCNN_OK;
}

// {d, heads, T, N} over rows of ld elements: a box of 64 tokens of one head, min(d, 64) columns wide
static int head_map(CUtensorMap *map, const void *base, const AttnShape &s) {
    const int boxc = s.d < 64 ? s.d : 64;
    const uint64_t dims[4] = {(uint64_t)s.d, (uint64_t)s.h, (uint64_t)s.T, (uint64_t)s.N};
    const uint64_t str[3] = {(uint64_t)s.d * 2, (uint64_t)s.ld * 2, (uint64_t)s.T * s.ld * 2};
    const uint32_t box[4] = {(uint32_t)boxc, 1, AT_ROWS, 1};
    const CUtensorMapSwizzle sw = boxc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : boxc == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
    return make_map_bf16(map, const_cast<void *>(base), 4, dims, str, box, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

// byte ranges [a, a + na) and [b, b + nb) intersect
static bool overlap(const void *a, size_t na, const void *b, size_t nb) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + nb && y < x + na;
}

// two outputs in rows of ldg elements, heads * d columns each: they may share a buffer on disjoint columns
static bool columns_clash(const void *a, const void *b, size_t bytes, long ldg, long hd) {
    if (!overlap(a, bytes, b, bytes)) return false;
    const long long delta = ((long long)(intptr_t)b - (long long)(intptr_t)a);
    if (delta % 2) return true;
    const long long r = ((delta / 2) % ldg + ldg) % ldg;
    return r < hd || r > ldg - hd;
}

static int launch(pcnn_ctx *ctx, int which, const AttnShape &s, const AttnMaps &m, const AttnParams &p) {
    const int grid = p.tiles < ctx->sm_count ? p.tiles : ctx->sm_count;
    void *args[] = {const_cast<AttnMaps *>(&m), const_cast<AttnParams *>(&p)};
    PCNN_CUDA(cudaLaunchKernel(variant(which, s.d), dim3((unsigned)grid), dim3(AT_THREADS), args,
                               (size_t)(which ? smem_bwd(s.d) : smem_fwd(s.d)), ctx->stream));
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

static bool misaligned(const void *p) { return ((uintptr_t)p & 15) != 0; }

extern "C" int pcnn_attention_bf16_fwd(pcnn_ctx *ctx, const void *q, const void *k, const void *v, int N, int T, int heads, int d, int ld,
                                       float scale, void *o, float *lse) {
    const char *fn = "pcnn_attention_bf16_fwd";
    PCNN_REQUIRE(ctx && q && k && v && o && lse, PCNN_ERR_ARG, "%s: NULL argument", fn);
    AttnShape s;
    int rc = attn_shape(fn, N, T, heads, d, ld, 0, scale, &s);
    if (rc) return rc;
    PCNN_REQUIRE(!misaligned(q) && !misaligned(k) && !misaligned(v) && !misaligned(o) && !misaligned(lse), PCNN_ERR_ARG,
                 "%s: q, k, v, o and lse must be 16-byte aligned", fn);
    const size_t nt = (size_t)N * T, hd = (size_t)heads * d;
    const size_t in_b = ((nt - 1) * ld + hd) * 2, o_b = nt * hd * 2, l_b = (size_t)N * heads * T * 4;
    PCNN_REQUIRE(!overlap(o, o_b, lse, l_b), PCNN_ERR_ARG, "%s: o and lse overlap", fn);
    for (const void *in : {q, k, v})
        PCNN_REQUIRE(!overlap(in, in_b, o, o_b) && !overlap(in, in_b, lse, l_b), PCNN_ERR_ARG, "%s: o or lse overlaps q, k or v", fn);
    pcnn_device_guard g(ctx->device);
    if ((rc = configure(ctx))) return rc;
    AttnMaps m;
    memset(&m, 0, sizeof(m));
    if ((rc = head_map(&m.q, q, s)) || (rc = head_map(&m.k, k, s)) || (rc = head_map(&m.v, v, s))) return rc;
    AttnParams p;
    memset(&p, 0, sizeof(p));
    p.T = T; p.h = heads; p.nblk = s.nblk; p.tiles = s.tiles; p.c2 = s.c2; p.scale = scale;
    p.o = static_cast<__nv_bfloat16 *>(o);
    p.lse = lse;
    return launch(ctx, 0, s, m, p);
}

extern "C" int pcnn_attention_bf16_bwd(pcnn_ctx *ctx, const void *q, const void *k, const void *v, const void *o, const void *dout,
                                       const float *lse, int N, int T, int heads, int d, int ld, float scale, void *dq, void *dk, void *dv,
                                       int ld_g) {
    const char *fn = "pcnn_attention_bf16_bwd";
    PCNN_REQUIRE(ctx && q && k && v && o && dout && lse && dq && dk && dv, PCNN_ERR_ARG, "%s: NULL argument", fn);
    AttnShape s;
    int rc = attn_shape(fn, N, T, heads, d, ld, ld_g, scale, &s);
    if (rc) return rc;
    PCNN_REQUIRE(!misaligned(q) && !misaligned(k) && !misaligned(v) && !misaligned(o) && !misaligned(dout) && !misaligned(lse) &&
                     !misaligned(dq) && !misaligned(dk) && !misaligned(dv),
                 PCNN_ERR_ARG, "%s: q, k, v, o, dout, lse, dq, dk and dv must be 16-byte aligned", fn);
    const size_t nt = (size_t)N * T, hd = (size_t)heads * d;
    const size_t in_b = ((nt - 1) * ld + hd) * 2, o_b = nt * hd * 2, l_b = (size_t)N * heads * T * 4, g_b = ((nt - 1) * ld_g + hd) * 2;
    const void *outs[3] = {dq, dk, dv};
    for (int a = 0; a < 3; ++a) {
        for (int b = a + 1; b < 3; ++b)
            PCNN_REQUIRE(!columns_clash(outs[a], outs[b], g_b, ld_g, (long)hd), PCNN_ERR_ARG,
                         "%s: dq, dk and dv may share a buffer only on disjoint columns of rows of ld_g elements", fn);
        for (const void *in : {q, k, v})
            PCNN_REQUIRE(!overlap(outs[a], g_b, in, in_b), PCNN_ERR_ARG, "%s: dq, dk or dv overlaps q, k or v", fn);
        PCNN_REQUIRE(!overlap(outs[a], g_b, o, o_b) && !overlap(outs[a], g_b, dout, o_b) && !overlap(outs[a], g_b, lse, l_b), PCNN_ERR_ARG,
                     "%s: dq, dk or dv overlaps o, dout or lse", fn);
    }
    pcnn_device_guard g(ctx->device);
    if ((rc = configure(ctx))) return rc;
    float *dsum = nullptr;
    if ((rc = pcnn_scratch(ctx, s.scratch, (void **)&dsum))) return rc;
    const long rows = (long)nt * heads;
    long blocks = (rows + 255) / 256;
    if (blocks > (long)ctx->sm_count * 8) blocks = (long)ctx->sm_count * 8;
    k_attn_dsum<<<(int)blocks, 256, 0, ctx->stream>>>(static_cast<const __nv_bfloat16 *>(o), static_cast<const __nv_bfloat16 *>(dout), dsum,
                                                      rows, T, heads, d);
    PCNN_CHECK_LAUNCH(ctx);
    AttnMaps m;
    memset(&m, 0, sizeof(m));
    AttnShape so = s;                       // o and dout are dense: rows of heads * d
    so.ld = (int)hd;
    if ((rc = head_map(&m.q, q, s)) || (rc = head_map(&m.k, k, s)) || (rc = head_map(&m.v, v, s)) || (rc = head_map(&m.dout, dout, so)))
        return rc;
    AttnParams p;
    memset(&p, 0, sizeof(p));
    p.T = T; p.h = heads; p.nblk = s.nblk; p.tiles = s.tiles; p.c2 = s.c2; p.scale = scale;
    p.lse_in = lse; p.dsum = dsum;
    p.dq = static_cast<__nv_bfloat16 *>(dq); p.dk = static_cast<__nv_bfloat16 *>(dk); p.dv = static_cast<__nv_bfloat16 *>(dv);
    p.ldg = ld_g;
    if ((rc = launch(ctx, 1, s, m, p))) return rc;
    return launch(ctx, 2, s, m, p);
}
