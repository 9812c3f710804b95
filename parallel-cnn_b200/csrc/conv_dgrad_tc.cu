// parallel-cnn_b200/csrc/conv_dgrad_tc.cu -- input gradient of the NHWC bf16 convolution (64 filters), row-streaming formulation.
//
//     dx[n][h][w][c] = sum_{k,r,s} dy[n][(h-r)/st][(w-s)/st][k] * f[k][r][s][c]     over the (r, s) with st | h-r, st | w-s
//
// (st = the window step of the forward, 1..4, a template parameter next to R, S, C; st = 1 is the reference's conv.)
//
// Access pattern first: every TMA box is a contiguous run of one dy row (pcnn_measure_tma_read mode 3 measures that pattern;
// mode 2, boxes gathering 128-byte pieces of different rows, is the alternative it was chosen over).
//   (More than 64 filters: K/64 channel groups per dy row -- K/64 x 4 boxes per stage and K/64 x 4 MMA steps per row; K <= 256.)
//   * A CTA owns a strip of <= 4 * st * (32 - FS) output columns (FS = (S-1) / st) and walks DOWN the rows of its share of
//     the images.  One dy row of the strip is an A operand [128 pixels x 64 channels] (4 boxes of <= 32 pixels, one per
//     lane quarter of oq output columns, oq a multiple of st; the box of a quarter starting at column w0 holds dy pixels
//     w0/st - FS .. (w0 + oq)/st - 1, so that the shift along s never crosses a quarter).
//   * Two warpgroups multiply it (64 pixels each) with a constant filter matrix whose N = NW columns are (r, s, c):
//     D[pixel][(r, s, c)] = sum_k dy[pixel][k] f[k][r][s][c], fresh for every dy row (wgmma, register accumulators).
//   * Rows are walked in units of st dx rows (U = ceil(H / st) per image); unit u reads dy row u when u < P, which
//     contributes to dx rows u*st .. u*st + R-1.  Each consumer thread owns a few (pixel, c) outputs of the strip and keeps
//     RR = st * ((R-1)/st + 1) partial rows of them in registers (a ring): after dy row u it adds
//     sum_s D[(l - s)/st + FS][(r, s, c)] (over the s with st | l - s) to partial row r of output column l, writes partial rows
//     0 .. st-1 (= dx rows u*st .. u*st + st-1, now complete; clipped at H) and shifts the ring by st rows.  Rows and columns
//     no window covers come out as zeros.  D passes through shared memory because the shift along s crosses the
//     accumulator's register layout.
//   * A CTA's share starts mid-image in general: the (R-1)/st dy rows above it are replayed and only the rows of the share
//     are written (0.5 % extra reads at config 5).
#include "tc_common.cuh"

#include <stdlib.h>

using namespace pcnn_tc;

namespace {

constexpr int D2_THREADS = 288;          // warps 0-7 two consumer warpgroups, warp 8 TMA producer
constexpr int D2_CONSUMERS = 256;
constexpr int D2_HALF_BYTES = 16384;     // one group of 64 channels: 4 quarters x 32 pixel rows x 128 B
constexpr int D2_MAX_STAGES = 11;
constexpr int D2_SMEM_BUDGET = 225 * 1024;

struct Dgrad2Params {
    int n_img, H, W, P, Q, U;            // U = ceil(H / st) row units per image
    int nstrips, strip_w, oq, bp;        // strips per row, output columns per strip / per lane quarter, pixels per TMA box
    int stages;                          // smem stages
    int KH;                              // channels / 64: a TMA box holds 64 channels (one 128-byte swizzle row per pixel)
    long long T;                         // n_img * U row units in walk order
    long long dx_pitch, dx_image_rows;
    __nv_bfloat16 *dx;
};

struct Dgrad2Ctl {
    unsigned long long full[D2_MAX_STAGES], empty[D2_MAX_STAGES], bfull;
};

// F[kh][n][kl] for column n = r * S * C + s * C + c: f[kh * 64 + kl][r][s][c], zero past R * S * C
__global__ void k_dgrad2_build_filter(const float *__restrict__ f, __nv_bfloat16 *__restrict__ T, int nw, int K, int R, int S, int C) {
    const int total = nw * K;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
        const int kl = idx % 64, n = (idx / 64) % nw, kh = idx / (64 * nw), k = kh * 64 + kl;
        float val = 0.0f;
        if (n < R * S * C) val = f[(long)k * R * S * C + n];
        T[idx] = __float2bfloat16_rn(val);
    }
}

// the row units one CTA walks, in order: (R-1)/st replayed units above its share, then its own units
struct RowWalk {
    long long t0, t1;       // share [t0, t1) of the walk
    __device__ RowWalk(const Dgrad2Params &p, int idx, int cnt) {
        const long long L = (p.T + cnt - 1) / cnt;
        t0 = (long long)idx * L;
        t1 = t0 + L < p.T ? t0 + L : p.T;
        if (t0 > t1) t0 = t1;
    }
};

template <int R, int S, int C, int ST> struct DgradShape {
    static constexpr int SC = S * C, NW = (R * SC + 15) / 16 * 16, DST = NW + 4;   // D staging row stride (floats)
    static constexpr int FS = (S - 1) / ST;                                        // dy pixels of a box left of its quarter
    static constexpr int LQ = 32 * ST;                                              // output-column slots per lane quarter
    static constexpr int ITEMS = (4 * LQ * C + D2_CONSUMERS - 1) / D2_CONSUMERS;   // (quarter, pixel, c) outputs per thread
    static constexpr int RR = ST * ((R - 1) / ST + 1);                              // partial dx rows in the ring
    static constexpr int NJ = (S + ST - 1) / ST;                                    // taps s = l % st + j * st, j < NJ
};

template <int R, int S, int C, int ST, int KHC>
__global__ void __launch_bounds__(D2_THREADS, 1)
k_conv_tc_dgrad_rows(const __grid_constant__ CUtensorMap map_dy, const __grid_constant__ CUtensorMap map_b, const Dgrad2Params p) {
    using SH = DgradShape<R, S, C, ST>;
    constexpr int SC = SH::SC, NW = SH::NW, DST = SH::DST, ITEMS = SH::ITEMS, FS = SH::FS, LQ = SH::LQ, RR = SH::RR, NJ = SH::NJ;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *base = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    constexpr int BMAT = NW * 128;
    // KHC > 0: the channel-group count is a compile-time constant; KHC = 0: p.KH groups at run time
    const int KH = KHC > 0 ? KHC : p.KH, STAGE = KH * D2_HALF_BYTES;
    unsigned char *bmat = base;                                         // [KH][NW][64] bf16, SWIZZLE_128B
    unsigned char *astage = base + (size_t)KH * BMAT;                   // [stages][KH][4][32][64] bf16, SWIZZLE_128B
    float *dst = reinterpret_cast<float *>(astage + (size_t)p.stages * STAGE);   // [128][DST] fp32
    Dgrad2Ctl &B = *reinterpret_cast<Dgrad2Ctl *>(dst + 128 * DST);
    const int NST = p.stages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // this CTA's strip of output columns and its share of the row walk
    const int strip = blockIdx.x % p.nstrips, idx = blockIdx.x / p.nstrips;
    const int cnt = ((int)gridDim.x - strip + p.nstrips - 1) / p.nstrips;
    const RowWalk walk(p, idx, cnt);
    const int w_strip = strip * p.strip_w;
    const int w_end = w_strip + p.strip_w < p.W ? w_strip + p.strip_w : p.W;
    const long long nel = walk.t1 - walk.t0;
    const int u_first = (int)(walk.t0 % p.U);
    const int n_first = (int)(walk.t0 / p.U);
    const int warm = u_first < (R - 1) / ST ? u_first : (R - 1) / ST;  // replayed units above the share (same image)
    const long long nrows = nel + warm;

    if (threadIdx.x == 0) {
        for (int i = 0; i < NST; ++i) { bar_init(&B.full[i], 1); bar_init(&B.empty[i], D2_CONSUMERS / 32); }
        bar_init(&B.bfull, 1);
        fence_barrier_init();
    }
    // pixel rows a box does not cover (box of bp < 32 pixels) must hold finite values: their D rows are never read
    for (int i = threadIdx.x * 16; i < NST * STAGE; i += D2_THREADS * 16) *reinterpret_cast<uint4 *>(astage + i) = make_uint4(0, 0, 0, 0);
    fence_proxy_async_smem();
    __syncthreads();
    if (nel <= 0) return;

    if (warp == D2_CONSUMERS / 32) {
        // ===== TMA producer =====
        if (lane == 0) {
            bar_expect_tx(&B.bfull, (unsigned)(KH * BMAT));
            for (int kh = 0; kh < KH; ++kh) tma_load_2d(bmat + (size_t)kh * BMAT, &map_b, 0, kh * NW, &B.bfull);
            int stage = 0;
            unsigned ph = 0;
            int n = n_first, u = u_first - warm;
            for (long long i = 0; i < nrows; ++i) {
                if (u < p.P) {
                    bar_wait_relaxed(&B.empty[stage], ph ^ 1u, 32);
                    bar_expect_tx(&B.full[stage], (unsigned)(KH * 4 * p.bp * 128));
                    unsigned char *a = astage + (size_t)stage * STAGE;
                    const int row = n * p.P + u;
                    for (int kh = 0; kh < KH; ++kh)
#pragma unroll
                        for (int g = 0; g < 4; ++g)      // pixels left of the image / right of its last dy pixel arrive as zeros
                            tma_load_3d(a + kh * D2_HALF_BYTES + g * 4096, &map_dy, kh * 64, (w_strip + g * p.oq) / ST - FS, row, &B.full[stage]);
                    if (++stage == NST) { stage = 0; ph ^= 1u; }
                }
                if (++u == p.U) { u = 0; ++n; }
            }
        }
        return;
    }

    // ===== consumers: D = dy row x F on the tensor cores, then the ring of partial dx rows in registers =====
    const int tid = threadIdx.x, wg = warp >> 2, wq = warp & 3;
    int it_q[ITEMS], it_l[ITEMS], it_c[ITEMS];
    bool it_ok[ITEMS];
    float ring[ITEMS][RR];
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
        const int item = tid + k * D2_CONSUMERS;
        it_q[k] = item / (LQ * C);
        it_l[k] = (item / C) % LQ;
        it_c[k] = item % C;
        int nvalid = w_end - (w_strip + it_q[k] * p.oq);
        if (nvalid > p.oq) nvalid = p.oq;
        it_ok[k] = item < 4 * LQ * C && it_l[k] < nvalid;
#pragma unroll
        for (int r = 0; r < RR; ++r) ring[k][r] = 0.0f;
    }
    bar_wait(&B.bfull, 0);
    const uint32_t b0 = s_u32(bmat), a_base = s_u32(astage) + (uint32_t)(wg * 64 * 128);
    int stage = 0;
    unsigned ph = 0;
    int n = n_first, u = u_first - warm;
    for (long long i = 0; i < nrows; ++i) {
        if (u < p.P) {
            float acc[NW / 2];
            bar_wait(&B.full[stage], ph);
            wg_fence();
            for (int kh = 0; kh < KH; ++kh) {          // 64 channels = 4 K steps of 16
                const uint32_t a0 = a_base + (uint32_t)(stage * STAGE + kh * D2_HALF_BYTES), bk = b0 + (uint32_t)(kh * BMAT);
#pragma unroll
                for (int ks = 0; ks < 4; ++ks)
                    wgmma_bf16<0, 0>(acc, gmma_desc_k_sw128(a0 + ks * 32), gmma_desc_k_sw128(bk + ks * 32), (kh | ks) != 0 ? 1u : 0u);
            }
            wg_commit();
            wg_wait<0>();
            wg_hold(acc);
            __syncwarp();
            if (lane == 0) bar_arrive(&B.empty[stage]);
            if (++stage == NST) { stage = 0; ph ^= 1u; }
#pragma unroll
            for (int j = 0; j < NW / 8; ++j)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int row = wg * 64 + wg_row(2 * hh, wq, lane), col = wg_col(4 * j, lane);
                    *reinterpret_cast<float2 *>(dst + row * DST + col) = make_float2(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]);
                }
            asm volatile("bar.sync 1, %0;" ::"n"(D2_CONSUMERS) : "memory");
#pragma unroll
            for (int k = 0; k < ITEMS; ++k) {
                // lane b of quarter g holds dy pixel w0/st - FS + b; output column l of the quarter needs, for each s with
                // st | l - s, dy pixel (w0 + l - s)/st, i.e. lane (l - s)/st + FS.  With s = l % st + j * st that is lane
                // (l - l % st)/st + FS - j.
                if (it_ok[k]) {
                    const int rl = ST == 1 ? 0 : it_l[k] % ST;
                    const float *d = dst + (it_q[k] * 32 + (it_l[k] - rl) / ST + FS) * DST + it_c[k];
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        float t = 0.0f;
#pragma unroll
                        for (int j = 0; j < NJ; ++j) {
                            const int s = rl + j * ST;
                            if (ST == 1 || s < S) t += d[-j * DST + r * SC + s * C];
                        }
                        ring[k][r] += t;
                    }
                }
            }
            asm volatile("bar.sync 1, %0;" ::"n"(D2_CONSUMERS) : "memory");   // D staging free for the next row
        }
        // dx rows u*st .. u*st + st-1 are complete (a later dy row starts at a later unit); units above the share are not
        // this CTA's
        if (i >= warm) {
#pragma unroll
            for (int v = 0; v < ST; ++v) {
                const int h = u * ST + v;
                if (ST == 1 || h < p.H) {
#pragma unroll
                    for (int k = 0; k < ITEMS; ++k)
                        if (it_ok[k])
                            p.dx[((long long)n * p.dx_image_rows + h) * p.dx_pitch + (long long)(w_strip + it_q[k] * p.oq + it_l[k]) * C + it_c[k]] =
                                __float2bfloat16_rn(ring[k][v]);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
#pragma unroll
            for (int r = 0; r + ST < RR; ++r) ring[k][r] = ring[k][r + ST];
#pragma unroll
            for (int r = RR - ST; r < RR; ++r) ring[k][r] = 0.0f;
        }
        if (++u == p.U) { u = 0; ++n; }
    }
}

// NW (filter-matrix columns) and the shared-memory bytes that do not depend on the stage count
struct Geometry { int nw; size_t fixed; };

Geometry geometry(int R, int S, int C, int KH) {
    Geometry g;
    g.nw = (R * S * C + 15) / 16 * 16;
    g.fixed = (size_t)KH * g.nw * 128 + (size_t)128 * (g.nw + 4) * 4 + sizeof(Dgrad2Ctl) + 1024;
    return g;
}

// column strips: strip width and lane-quarter width oq are multiples of st, oq <= st * (32 - FS) so that a quarter's box of
// oq/st + FS dy pixels fits the 32 pixel rows of a quarter
struct Strips { int nstrips, strip_w, oq, bp; };

Strips strips(int W, int S, int st) {
    Strips t;
    const int fs = (S - 1) / st, oq_max = st * (32 - fs);
    t.nstrips = (W + 4 * oq_max - 1) / (4 * oq_max);
    t.strip_w = ((W + t.nstrips - 1) / t.nstrips + st - 1) / st * st;
    t.oq = ((t.strip_w + 3) / 4 + st - 1) / st * st;
    t.bp = t.oq / st + fs;
    return t;
}

template <int R, int S, int C, int ST, int KHC>
int launch_rows_k(pcnn_ctx *ctx, const CUtensorMap &map_dy, const CUtensorMap &map_b, const Dgrad2Params &p, int grid, size_t smem) {
    static bool configured[64] = {};        // function attributes are per device
    if (!configured[ctx->device & 63]) {
        PCNN_CUDA(cudaFuncSetAttribute(k_conv_tc_dgrad_rows<R, S, C, ST, KHC>, cudaFuncAttributeMaxDynamicSharedMemorySize, D2_SMEM_BUDGET + 2048));
        configured[ctx->device & 63] = true;
    }
    k_conv_tc_dgrad_rows<R, S, C, ST, KHC><<<grid, D2_THREADS, smem, ctx->stream>>>(map_dy, map_b, p);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
template <int R, int S, int C, int ST>
int launch_rows(pcnn_ctx *ctx, const CUtensorMap &map_dy, const CUtensorMap &map_b, const Dgrad2Params &p, int grid, size_t smem) {
    return p.KH == 1 ? launch_rows_k<R, S, C, ST, 1>(ctx, map_dy, map_b, p, grid, smem) : launch_rows_k<R, S, C, ST, 0>(ctx, map_dy, map_b, p, grid, smem);
}

// the instantiated (R, S, C, st): stride 1 and 2 for every (R, S, C) below, strides 3 and 4 for 3x3 with C <= 3
bool instantiated(int R, int S, int C, int st) {
    const bool small = R == 3 && S == 3 && (C == 1 || C == 2 || C == 3);
    const bool any = small || (R == 3 && S == 3 && (C == 4 || C == 8)) || (R == 5 && S == 5 && (C == 1 || C == 3)) || (R == 7 && S == 7 && C == 1);
    return st <= 2 ? any : st <= 4 && small;
}

template <int ST>
int launch_stride(pcnn_ctx *ctx, const CUtensorMap &map_dy, const CUtensorMap &map_b, const Dgrad2Params &p, int grid, size_t smem, int R, int S, int C) {
    if (R == 3 && S == 3 && C == 3) return launch_rows<3, 3, 3, ST>(ctx, map_dy, map_b, p, grid, smem);
    if (R == 3 && S == 3 && C == 1) return launch_rows<3, 3, 1, ST>(ctx, map_dy, map_b, p, grid, smem);
    if (R == 3 && S == 3 && C == 2) return launch_rows<3, 3, 2, ST>(ctx, map_dy, map_b, p, grid, smem);
    if constexpr (ST <= 2) {
        if (R == 3 && S == 3 && C == 4) return launch_rows<3, 3, 4, ST>(ctx, map_dy, map_b, p, grid, smem);
        if (R == 5 && S == 5 && C == 1) return launch_rows<5, 5, 1, ST>(ctx, map_dy, map_b, p, grid, smem);
        if (R == 3 && S == 3 && C == 8) return launch_rows<3, 3, 8, ST>(ctx, map_dy, map_b, p, grid, smem);
        if (R == 5 && S == 5 && C == 3) return launch_rows<5, 5, 3, ST>(ctx, map_dy, map_b, p, grid, smem);
        if (R == 7 && S == 7 && C == 1) return launch_rows<7, 7, 1, ST>(ctx, map_dy, map_b, p, grid, smem);
    }
    pcnn_set_error("pcnn_conv_dgrad: no row-streaming instantiation for R = %d, S = %d, C = %d, stride %d", R, S, C, ST);
    return PCNN_ERR_ARG;
}

}  // namespace

bool pcnn_conv_dgrad_rows_ok(int N, int H, int W, int C, int K, int R, int S, int st, const void *dy) {
    if (K % 64 || K > 256 || ((uintptr_t)dy & 15) || N <= 0 || H < R || W < S) return false;
    if (!instantiated(R, S, C, st)) return false;
    const Geometry g = geometry(R, S, C, K / 64);
    return g.nw <= 256 && S <= 16 && g.fixed + 2 * (size_t)(K / 64) * D2_HALF_BYTES <= (size_t)D2_SMEM_BUDGET;
}

// host-side tiling of the row-streaming input gradient, for pcnn_conv_bwd_plan_info (no GPU needed)
void pcnn_conv_dgrad_rows_info(int H, int W, int C, int K, int R, int S, int st, int *out4) {
    const Geometry g = geometry(R, S, C, K / 64);
    const Strips t = strips(W, S, st);
    const size_t stage_bytes = (size_t)(K / 64) * D2_HALF_BYTES;
    int ns = stage_bytes ? (int)(((size_t)D2_SMEM_BUDGET - g.fixed) / stage_bytes) : 0;
    out4[0] = t.nstrips; out4[1] = t.oq; out4[2] = st * ((R - 1) / st + 1); out4[3] = ns > D2_MAX_STAGES ? D2_MAX_STAGES : ns;
    (void)H;
}

// dy_channels: as for pcnn_conv_wgrad_rows (filters dy really holds; the TMA zero-fills the rest of a 64-channel box)
int pcnn_conv_dgrad_rows(pcnn_ctx *ctx, const void *dy_bf16, const float *filt_f32_dev, void *dx_bf16, int N, int H, int W, int C, int K,
                         int R, int S, int st, int row_pitch, int image_rows, int dy_channels) {
    const uint64_t KD = dy_channels > 0 ? (uint64_t)dy_channels : (uint64_t)K;
    pcnn_device_guard guard(ctx->device);
    const Geometry g = geometry(R, S, C, K / 64);
    Dgrad2Params p;
    memset(&p, 0, sizeof(p));
    p.n_img = N; p.H = H; p.W = W; p.P = (H - R) / st + 1; p.Q = (W - S) / st + 1; p.U = (H + st - 1) / st;
    const Strips t = strips(W, S, st);
    p.nstrips = t.nstrips; p.strip_w = t.strip_w; p.oq = t.oq; p.bp = t.bp;
    p.T = (long long)N * p.U;
    p.dx_pitch = row_pitch > 0 ? row_pitch : W * C;
    p.dx_image_rows = image_rows > 0 ? image_rows : H;
    p.dx = reinterpret_cast<__nv_bfloat16 *>(dx_bf16);
    p.KH = K / 64;
    const size_t stage_bytes = (size_t)p.KH * D2_HALF_BYTES;
    const int ns = (int)(((size_t)D2_SMEM_BUDGET - g.fixed) / stage_bytes);
    p.stages = ns > D2_MAX_STAGES ? D2_MAX_STAGES : ns;
    PCNN_REQUIRE(p.stages >= 2, PCNN_ERR_ARG, "pcnn_conv_dgrad: the filter matrix leaves no room for two stages");
    const size_t smem = g.fixed + (size_t)p.stages * stage_bytes;

    __nv_bfloat16 *T = nullptr;
    const size_t t_elems = (size_t)g.nw * K;
    int rc = pcnn_scratch(ctx, t_elems * 2, (void **)&T);
    if (rc) return rc;
    k_dgrad2_build_filter<<<(int)((t_elems + 255) / 256), 256, 0, ctx->stream>>>(filt_f32_dev, T, g.nw, K, R, S, C);
    PCNN_CHECK_LAUNCH(ctx);

    CUtensorMap map_dy, map_b;
    {
        const uint64_t dims[3] = {KD, (uint64_t)p.Q, (uint64_t)N * p.P};
        const uint64_t str[2] = {KD * 2, (uint64_t)p.Q * KD * 2};
        const uint32_t box[3] = {64, (uint32_t)p.bp, 1};
        if ((rc = make_map_bf16(&map_dy, const_cast<void *>(dy_bf16), 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B)))
            return rc;
        const uint64_t bd[2] = {64, (uint64_t)p.KH * g.nw};            // [channel group][nw] rows of 64 channels
        const uint64_t bs[1] = {128};
        const uint32_t bb[2] = {64, (uint32_t)g.nw};
        if ((rc = make_map_bf16(&map_b, T, 2, bd, bs, bb, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B))) return rc;
    }
    // every CTA needs at least one row of its strip; more CTAs than rows would leave empty shares (handled, but pointless)
    long long want = p.T * p.nstrips;
    const int grid = (int)(want < ctx->sm_count ? want : ctx->sm_count);
    switch (st) {
        case 1: return launch_stride<1>(ctx, map_dy, map_b, p, grid, smem, R, S, C);
        case 2: return launch_stride<2>(ctx, map_dy, map_b, p, grid, smem, R, S, C);
        case 3: return launch_stride<3>(ctx, map_dy, map_b, p, grid, smem, R, S, C);
        case 4: return launch_stride<4>(ctx, map_dy, map_b, p, grid, smem, R, S, C);
    }
    pcnn_set_error("pcnn_conv_dgrad: stride %d outside 1..4", st);
    return PCNN_ERR_ARG;
}
