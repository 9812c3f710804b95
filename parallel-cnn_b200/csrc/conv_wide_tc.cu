// parallel-cnn_b200/csrc/conv_wide_tc.cu -- bf16 convolution forward for wide channel counts on the Hopper tensor cores
// (pcnn_conv_wide_plan_create): the shapes the row-Toeplitz forward of conv_tc.cu refuses, C % 8 == 0, K <= 256.
//
// Formulation ("tap-major implicit GEMM").  With M = output pixels, N = filters and the reduction over (r, s, c):
//     y[n][p][q][k] = sum_{r,s}  sum_c  x[n][p*st + r][q*st + s][c] * f[k][r][s][c]
// i.e. R*S GEMMs whose A operand is the input shifted by the tap (r, s) and whose B operand is the filter slice f[:, r, s, :].
// The reduction runs in steps of 64 channels (one 128-byte SWIZZLE_128B row per pixel / filter), R*S*ceil(C/64) steps per
// tile, four m64nNk16 per step and warpgroup.  Nothing is expanded in memory:
//   * A: a tile is a Pt x Qt block of output pixels of one image (Pt * Qt = 128).  For tap (r, s) the block reads one TMA box
//     {64 channels, Qt, Pt, 1} of the map of x that starts at input row r % st and column s % st and steps st rows and st
//     pixels (one map per such phase, at most st^2 = 16): box coordinate (q0 + s / st, p0 + r / st) is then input pixel
//     ((p0 + pp) * st + r, (q0 + qq) * st + s) for the block's pixel (pp, qq).  The map extents stop at the last row / pixel of
//     the image and at channel C: everything outside is zero-filled, pad rows and columns of x are never read.
//   * B: the filters rounded to bf16 on the device (at creation and by pcnn_conv_plan_set_params), KRSC, viewed as {C, R*S, K}: a box {64, 1, Npad} is the K-major
//     operand of one step; channels >= C and filters >= K are zero-filled by TMA, and a box never reaches the next tap.
//   * D: [128 x Npad] fp32 in the registers of two warpgroups (rows 0-63 / 64-127 of the block), Npad = K rounded up to 16.
//   * Epilogue: bias, activation (none, sigmoid or ReLU), bf16, written to a shared staging tile per warpgroup (SWIZZLE_128B,
//     conflict-free), then stored by TMA through a map of y {K, Q, P, N} that clips pixels outside the image and channels >= K.  The store
//     drains while the warpgroup already runs the next tile's MMAs; the staging tile is reused once its store has been read.
// Pixel blocks on small images issue more pixels than they compute: pcnn_conv_wide_plan_info reports both.
//
// Zero padding (pcnn_conv_wide_plan_create_padded) moves the box coordinates only: with r - pad_h = st * a_r + rho_r (floor
// division, 0 <= rho_r < st) tap r reads phase map rho_r at box row p0 + a_r, and columns the same (ConvWideTaps).  A box row
// or column before the image (a_r < 0) or past it is zero-filled by TMA like the channels >= C; nothing else changes.
// Dilation (pcnn_conv_wide_plan_create_dilated) is the same table with r * dil_h - pad_h in place of r - pad_h: the device code is
// the padded forward's, unchanged.
//
// Warp roles (288 threads, 1 CTA/SM, persistent over tiles): warps 0-7 = two consumer warpgroups, warp 8 = TMA producer.
#include "tc_common.cuh"

#include <memory>

using namespace pcnn_tc;

namespace {

constexpr int WD_THREADS = 288;
constexpr int WD_CONSUMER_WARPS = 8;
constexpr int WD_M = 128;                 // output pixels per tile (two warpgroups of 64)
constexpr int WD_KC = 64;                 // channels per reduction step (128 B rows, SWIZZLE_128B)
constexpr int WD_MAX_STAGES = 8;
constexpr int WD_SMEM_BUDGET = 225 * 1024;
constexpr int WD_A_BYTES = WD_M * WD_KC * 2;       // 16 KB
constexpr int WD_STG_BYTES = 64 * WD_KC * 2;       // one staging sub-tile: 64 pixels x 64 channels, 8 KB
constexpr int WD_MAX_RS = 7;
constexpr int WD_MAX_DIL = 256;

struct ConvWideParams {
    int Pt, Qt;                  // pixel block: Pt output rows x Qt output columns
    int n_pb, n_qb, tiles;       // blocks per image column / row, N * n_pb * n_qb
    int R, S, stride, nch;       // taps, window step, 64-channel chunks per tap
    int stages, K;
    const float *bias;           // [K] or null
    ConvWideTaps taps;           // x phase and box offset of every tap row / column
};

struct ConvWideMaps {
    CUtensorMap x[16];           // phase (rph[r], sph[s]) at index rph[r] * st + sph[s]
    CUtensorMap w;               // filters {C, R*S, K}
    CUtensorMap y;               // output {K, Q, P, N}
};

struct ConvWideCtl {
    float bias[256];
    unsigned long long full[WD_MAX_STAGES], empty[WD_MAX_STAGES];
};

// dynamic shared memory, 1024-byte aligned: [2 x nsub staging sub-tiles] [stages x (A tile, B tile)] [ctl]
static size_t wide_stage_bytes(int npad) { return (size_t)WD_A_BYTES + (size_t)npad * WD_KC * 2; }
static size_t wide_staging_bytes(int npad) { return 2 * (size_t)((npad + 63) / 64) * WD_STG_BYTES; }
static size_t wide_smem_bytes(int npad, int stages) {
    return wide_staging_bytes(npad) + (size_t)stages * wide_stage_bytes(npad) + sizeof(ConvWideCtl) + 1024;
}

template <int ACT, int N>
__global__ void __launch_bounds__(WD_THREADS, 1)
k_conv_wide_fwd(const __grid_constant__ ConvWideMaps m, const ConvWideParams p) {
    constexpr int NSUB = (N + 63) / 64;
    constexpr int B_BYTES = N * WD_KC * 2;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *base = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    unsigned char *stg = base;
    unsigned char *ring = base + 2 * NSUB * WD_STG_BYTES;
    const int NST = p.stages;
    ConvWideCtl &S = *reinterpret_cast<ConvWideCtl *>(ring + (size_t)NST * (WD_A_BYTES + B_BYTES));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nsteps = p.R * p.S * p.nch;

    if (threadIdx.x == 0) {
        for (int i = 0; i < NST; ++i) { bar_init(&S.full[i], 1); bar_init(&S.empty[i], WD_CONSUMER_WARPS); }
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < 256; i += WD_THREADS) S.bias[i] = (p.bias && i < p.K) ? p.bias[i] : 0.0f;
    __syncthreads();

    if (warp == WD_CONSUMER_WARPS) {
        // ===== TMA producer: per tile and step one box of x and one box of filters =====
        if (lane == 0) {
            int it = 0;
            for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
                const int n = tile / (p.n_pb * p.n_qb), rem = tile % (p.n_pb * p.n_qb);
                const int p0 = (rem / p.n_qb) * p.Pt, q0 = (rem % p.n_qb) * p.Qt;
                for (int r = 0; r < p.R; ++r)
                    for (int s = 0; s < p.S; ++s) {
                        const CUtensorMap *mx = &m.x[p.taps.rph[r] * p.stride + p.taps.sph[s]];
                        const int bq = q0 + p.taps.soff[s], bp = p0 + p.taps.roff[r];
                        for (int ch = 0; ch < p.nch; ++ch, ++it) {
                            const int stage = it % NST;
                            const unsigned ph = (unsigned)(it / NST) & 1u;
                            bar_wait_relaxed(&S.empty[stage], ph ^ 1u, 32);
                            unsigned char *a = ring + (size_t)stage * (WD_A_BYTES + B_BYTES);
                            bar_expect_tx(&S.full[stage], (unsigned)(WD_A_BYTES + B_BYTES));
                            tma_load_4d(a, mx, ch * WD_KC, bq, bp, n, &S.full[stage]);
                            tma_load_3d(a + WD_A_BYTES, &m.w, ch * WD_KC, r * p.S + s, 0, &S.full[stage]);
                        }
                    }
            }
        }
        return;
    }

    // ===== consumer warpgroups: MMA into registers, then bias / activation -> bf16 -> staging -> TMA store =====
    const int wg = warp >> 2, wq = warp & 3;
    const int tid_wg = threadIdx.x & 127;
    unsigned char *my_stg = stg + (size_t)wg * NSUB * WD_STG_BYTES;
    const uint32_t stg_s = s_u32(my_stg), bias_s = s_u32(S.bias);
    // the warpgroup's half of the block: rows pp in [wg * Pt/2, +Pt/2) of the block, or columns [wg * 64, +64) when Pt = 1
    const int dp = p.Pt >= 2 ? wg * (p.Pt / 2) : 0, dq = p.Pt >= 2 ? 0 : wg * 64;
    int it = 0;
    for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
        float acc[N / 2];
        for (int step = 0; step < nsteps; ++step, ++it) {
            const int stage = it % NST;
            bar_wait(&S.full[stage], (unsigned)(it / NST) & 1u);
            const uint32_t a0 = s_u32(ring + (size_t)stage * (WD_A_BYTES + B_BYTES)) + (uint32_t)(wg * 64 * WD_KC * 2);
            const uint32_t b0 = s_u32(ring + (size_t)stage * (WD_A_BYTES + B_BYTES) + WD_A_BYTES);
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < WD_KC / 16; ++ks)       // K = 16 bf16 = 32 bytes per instruction
                wgmma_bf16<0, 0>(acc, gmma_desc_k_sw128(a0 + ks * 32), gmma_desc_k_sw128(b0 + ks * 32), (step | ks) != 0 ? 1u : 0u);
            wg_commit();
            if (step > 0) {                               // the previous step's MMAs have retired: its stage is free
                wg_wait<1>();
                __syncwarp();
                if (lane == 0) bar_arrive(&S.empty[(it - 1) % NST]);
            }
        }
        wg_wait<0>();
        wg_hold(acc);
        __syncwarp();
        if (lane == 0) bar_arrive(&S.empty[(it - 1) % NST]);

        // the previous tile's stores have read the staging tile
        if (tid_wg == 0) bulk_wait_read0();
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = wg_row(2 * h, wq, lane);      // pixel of the warpgroup's half, 0..63
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                const int c = wg_col(4 * j, lane);
                float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
                float2 bb;
                asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(bb.x), "=f"(bb.y) : "r"(bias_s + (uint32_t)c * 4u));
                f0 += bb.x; f1 += bb.y;
                f0 = apply_act<ACT>(f0); f1 = apply_act<ACT>(f1);
                __nv_bfloat162 v = __floats2bfloat162_rn(f0, f1);
                // sub-tile j / 8 holds channels 64 (j / 8) ..; 16-byte chunk j % 8 of the row, XOR-swizzled by row % 8 (SWIZZLE_128B)
                const uint32_t addr = stg_s + (uint32_t)((j / 8) * WD_STG_BYTES + row * 128 + (((j % 8) ^ (row & 7)) << 4) + (lane & 3) * 4);
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(*reinterpret_cast<uint32_t *>(&v)) : "memory");
            }
        }
        fence_proxy_async_smem();
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
        if (tid_wg == 0) {
            const int n = tile / (p.n_pb * p.n_qb), rem = tile % (p.n_pb * p.n_qb);
            const int p0 = (rem / p.n_qb) * p.Pt, q0 = (rem % p.n_qb) * p.Qt;
#pragma unroll
            for (int sub = 0; sub < NSUB; ++sub) tma_store_4d(&m.y, my_stg + sub * WD_STG_BYTES, sub * 64, q0 + dq, p0 + dp, n);
            bulk_commit();
        }
    }
    if (tid_wg == 0) bulk_wait0();
}

typedef void (*conv_wide_fn)(const ConvWideMaps, const ConvWideParams);
#define PCNN_WIDE_ROW(N) \
    {k_conv_wide_fwd<PCNN_ACT_NONE, N>, k_conv_wide_fwd<PCNN_ACT_SIGMOID, N>, k_conv_wide_fwd<PCNN_ACT_RELU, N>}
static const void *conv_wide_variant(int act, int npad) {
    static const conv_wide_fn table[16][3] = {
        PCNN_WIDE_ROW(16),  PCNN_WIDE_ROW(32),  PCNN_WIDE_ROW(48),  PCNN_WIDE_ROW(64),  PCNN_WIDE_ROW(80),  PCNN_WIDE_ROW(96),
        PCNN_WIDE_ROW(112), PCNN_WIDE_ROW(128), PCNN_WIDE_ROW(144), PCNN_WIDE_ROW(160), PCNN_WIDE_ROW(176), PCNN_WIDE_ROW(192),
        PCNN_WIDE_ROW(208), PCNN_WIDE_ROW(224), PCNN_WIDE_ROW(240), PCNN_WIDE_ROW(256)};
    return reinterpret_cast<const void *>(table[npad / 16 - 1][pcnn_act_col(act)]);
}
#undef PCNN_WIDE_ROW

}  // namespace

// The pixel block of a P x Q output image: the Pt x Qt = 128 split that issues the fewest pixels; ties go to the wider block
// (longer contiguous rows).  Returns the blocks per image.
long long conv_wide_pixel_block(int P, int Q, int *Pt, int *Qt) {
    long long best = -1;
    for (int qt = 128; qt >= 1; qt /= 2) {
        const int pt = WD_M / qt;
        const long long blocks = (long long)((P + pt - 1) / pt) * ((Q + qt - 1) / qt);
        if (best < 0 || blocks < best) { best = blocks; *Pt = pt; *Qt = qt; }
    }
    return best;
}

// r * dil - pad = st * off[r] + ph[r], 0 <= ph[r] < st (floor division: r * dil - pad >= -pad may lie many strides before 0)
static void wide_tap_table(int R, int pad, int dil, int st, int *ph, int *off) {
    for (int r = 0; r < R; ++r) {
        const int t = r * dil - pad;
        ph[r] = ((t % st) + st) % st;
        off[r] = (t - ph[r]) / st;
    }
}

int conv_wide_shape(const char *fn, int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w, int dil_h,
                    int dil_w, int row_pitch, int image_rows, ConvWideShape *out) {
    PCNN_REQUIRE(stride >= 1 && stride <= 4, PCNN_ERR_ARG, "%s: stride %d outside 1..4", fn, stride);
    PCNN_REQUIRE(R >= 1 && R <= WD_MAX_RS && S >= 1 && S <= WD_MAX_RS, PCNN_ERR_ARG,
                 "%s: R = %d, S = %d: taps must be 1..7 in each direction", fn, R, S);
    PCNN_REQUIRE(dil_h >= 1 && dil_h <= WD_MAX_DIL && dil_w >= 1 && dil_w <= WD_MAX_DIL, PCNN_ERR_ARG,
                 "%s: dilation (%d, %d): 1 <= dil_h, dil_w <= %d are required", fn, dil_h, dil_w, WD_MAX_DIL);
    const bool dilated = dil_h > 1 || dil_w > 1;
    const int Eh = dil_h * (R - 1) + 1, Ew = dil_w * (S - 1) + 1;     // the window's extent
    if (!dilated)
        PCNN_REQUIRE(pad_h >= 0 && pad_h < R && pad_w >= 0 && pad_w < S, PCNN_ERR_ARG,
                     "%s: padding (%d, %d) with R = %d, S = %d taps: 0 <= pad_h <= R - 1 and 0 <= pad_w <= S - 1 are required", fn, pad_h,
                     pad_w, R, S);
    else
        PCNN_REQUIRE(pad_h >= 0 && pad_h < Eh && pad_w >= 0 && pad_w < Ew, PCNN_ERR_ARG,
                     "%s: padding (%d, %d) with R = %d, S = %d taps at dilation (%d, %d): 0 <= pad_h <= dil_h*(R - 1) and "
                     "0 <= pad_w <= dil_w*(S - 1) are required", fn, pad_h, pad_w, R, S, dil_h, dil_w);
    const bool padded = pad_h > 0 || pad_w > 0;
    if (dilated)
        PCNN_REQUIRE(N > 0 && H >= Eh - 2 * pad_h && W >= Ew - 2 * pad_w && C > 0 && K > 0, PCNN_ERR_ARG,
                     "%s: bad shape N=%d H=%d W=%d C=%d K=%d R=%d S=%d padding (%d, %d) dilation (%d, %d): H + 2*pad_h >= dil_h*(R - 1) + 1 "
                     "and W + 2*pad_w >= dil_w*(S - 1) + 1 are required", fn, N, H, W, C, K, R, S, pad_h, pad_w, dil_h, dil_w);
    else if (!padded)
        PCNN_REQUIRE(N > 0 && H >= R && W >= S && C > 0 && K > 0, PCNN_ERR_ARG,
                     "%s: bad shape N=%d H=%d W=%d C=%d K=%d R=%d S=%d", fn, N, H, W, C, K, R, S);
    else
        PCNN_REQUIRE(N > 0 && H >= R - 2 * pad_h && W >= S - 2 * pad_w && C > 0 && K > 0, PCNN_ERR_ARG,
                     "%s: bad shape N=%d H=%d W=%d C=%d K=%d R=%d S=%d padding (%d, %d): H + 2*pad_h >= R and W + 2*pad_w >= S are "
                     "required", fn, N, H, W, C, K, R, S, pad_h, pad_w);
    // a padded direction may read any phase of x (some tap lands on each residue (r*dil - pad) mod st): each must have a row /
    // pixel inside the image.  Unpadded, the phases read are (r*dil) mod st <= (E - 1) mod st, inside the image since H >= E.
    PCNN_REQUIRE((pad_h == 0 || H >= stride) && (pad_w == 0 || W >= stride), PCNN_ERR_ARG,
                 "%s: H = %d, W = %d with padding (%d, %d) at stride %d: a padded direction needs at least stride rows / pixels, "
                 "so that every phase of x has one inside the image", fn, H, W, pad_h, pad_w, stride);
    PCNN_REQUIRE(K % 8 == 0 && K <= 256, PCNN_ERR_ARG,
                 "%s: K = %d filters: K %% 8 == 0 and K <= 256 are required", fn, K);
    PCNN_REQUIRE(C % 8 == 0, PCNN_ERR_ARG,
                 "%s: C = %d channels: C %% 8 == 0 is required (16-byte pixel stride of the TMA map)", fn, C);
    PCNN_REQUIRE(row_pitch >= W * C && row_pitch % 8 == 0, PCNN_ERR_ARG,
                 "%s: row pitch %d must be >= W*C and a multiple of 8 elements (TMA 16-byte strides)", fn, row_pitch);
    if (image_rows <= 0) image_rows = H;
    PCNN_REQUIRE(image_rows >= H, PCNN_ERR_ARG, "%s: image pitch of %d rows is smaller than H = %d", fn, image_rows, H);
    int tc[5];                              // the row-Toeplitz plan has no padding and no dilation: such a shape is this plan's alone
    PCNN_REQUIRE(padded || dilated || pcnn_conv_tc_plan_info(N, H, W, C, K, R, S, stride, row_pitch, image_rows, tc) != PCNN_OK,
                 PCNN_ERR_ARG, "%s: this shape is served by the row-Toeplitz forward: use pcnn_conv_tc_plan_create", fn);
    const int P = (H + 2 * pad_h - Eh) / stride + 1, Q = (W + 2 * pad_w - Ew) / stride + 1;
    const long long best = conv_wide_pixel_block(P, Q, &out->Pt, &out->Qt);
    out->n_pb = (P + out->Pt - 1) / out->Pt;
    out->n_qb = (Q + out->Qt - 1) / out->Qt;
    PCNN_REQUIRE((long long)N * best < (1LL << 31), PCNN_ERR_ARG, "%s: %lld tiles exceed the int range", fn, (long long)N * best);
    out->tiles = (int)(N * best);
    out->nch = (C + WD_KC - 1) / WD_KC;
    out->npad = (K + 15) / 16 * 16;
    const size_t fixed = wide_smem_bytes(out->npad, 0);
    int st = (int)(((size_t)WD_SMEM_BUDGET - fixed) / wide_stage_bytes(out->npad));
    out->stages = st > WD_MAX_STAGES ? WD_MAX_STAGES : st;
    out->P = P; out->Q = Q;
    wide_tap_table(R, pad_h, dil_h, stride, out->taps.rph, out->taps.roff);
    wide_tap_table(S, pad_w, dil_w, stride, out->taps.sph, out->taps.soff);
    return PCNN_OK;
}

// x phase (rb, sb) of the window step: input rows rb, rb + st, ... and pixels sb, sb + st, ... of every image; the extents end at
// the image's last row and pixel, so a box never reads pad rows, pad columns or the next image.  Only the phases some tap reads
// are encoded (rb < min(st, R) at pad 0; with padding they need not be a prefix); each has a row and a pixel inside the image
// (H >= dil_h*(R - 1) + 1 at pad 0, H >= st when padded, and the same for W).
int conv_wide_x_maps(CUtensorMap *maps, const void *x_bf16, int N, int H, int W, int C, int R, int S, int st, const ConvWideTaps &taps,
                     int row_pitch, int image_rows, int Pt, int Qt) {
    bool row_used[4] = {}, col_used[4] = {};
    for (int r = 0; r < R; ++r) row_used[taps.rph[r]] = true;
    for (int s = 0; s < S; ++s) col_used[taps.sph[s]] = true;
    for (int rb = 0; rb < st; ++rb)
        for (int sb = 0; sb < st; ++sb) {
            if (!row_used[rb] || !col_used[sb]) continue;
            const uint64_t dims[4] = {(uint64_t)C, (uint64_t)((W - sb + st - 1) / st), (uint64_t)((H - rb + st - 1) / st), (uint64_t)N};
            const uint64_t str[3] = {(uint64_t)st * C * 2, (uint64_t)st * row_pitch * 2, (uint64_t)image_rows * row_pitch * 2};
            const uint32_t box[4] = {WD_KC, (uint32_t)Qt, (uint32_t)Pt, 1};
            void *base = const_cast<char *>(static_cast<const char *>(x_bf16)) + ((size_t)rb * row_pitch + (size_t)sb * C) * 2;
            int rc = make_map_bf16(&maps[rb * st + sb], base, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
            if (rc) return rc;
        }
    return PCNN_OK;
}

// a plan of pcnn_conv_wide_plan_create(_padded, _dilated): w is [K][R*S*C], the KRSC master with rows of R*S*C elements and no pad
struct ConvWidePlan : pcnn_conv_plan {
    ConvWideParams p;
    ConvWideShape sh;
    int N, H, W, C, row_pitch, image_rows, act;
    CUtensorMap map_w;
    int fwd(pcnn_ctx *ctx, const void *x_bf16, void *y_bf16) override;
};

// the query of the create call `fn` (its refusals name that call)
static int wide_plan_info(const char *fn, int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w,
                          int dil_h, int dil_w, int row_pitch, int image_rows, int *out8) {
    ConvWideShape sh;
    int rc = conv_wide_shape(fn, N, H, W, C, K, R, S, stride, pad_h, pad_w, dil_h, dil_w, row_pitch, image_rows, &sh);
    if (rc) return rc;
    out8[0] = sh.Pt; out8[1] = sh.Qt; out8[2] = sh.nch; out8[3] = sh.stages;
    out8[4] = sh.tiles; out8[5] = sh.n_pb; out8[6] = sh.n_qb; out8[7] = sh.npad;
    return PCNN_OK;
}

extern "C" int pcnn_conv_wide_plan_info(int N, int H, int W, int C, int K, int R, int S, int stride, int row_pitch, int image_rows,
                                        int *out8) {
    PCNN_REQUIRE(out8, PCNN_ERR_ARG, "pcnn_conv_wide_plan_info: NULL argument");
    return wide_plan_info("pcnn_conv_wide_plan_create", N, H, W, C, K, R, S, stride, 0, 0, 1, 1, row_pitch, image_rows, out8);
}

extern "C" int pcnn_conv_wide_plan_info_padded(int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w,
                                               int row_pitch, int image_rows, int *out8) {
    PCNN_REQUIRE(out8, PCNN_ERR_ARG, "pcnn_conv_wide_plan_info_padded: NULL argument");
    return wide_plan_info("pcnn_conv_wide_plan_create_padded", N, H, W, C, K, R, S, stride, pad_h, pad_w, 1, 1, row_pitch, image_rows,
                          out8);
}

extern "C" int pcnn_conv_wide_plan_info_dilated(int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w,
                                                int dil_h, int dil_w, int row_pitch, int image_rows, int *out8) {
    PCNN_REQUIRE(out8, PCNN_ERR_ARG, "pcnn_conv_wide_plan_info_dilated: NULL argument");
    return wide_plan_info("pcnn_conv_wide_plan_create_dilated", N, H, W, C, K, R, S, stride, pad_h, pad_w, dil_h, dil_w, row_pitch,
                          image_rows, out8);
}

static int wide_plan_create(const char *fn, pcnn_ctx *ctx, int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h,
                            int pad_w, int dil_h, int dil_w, int row_pitch, int image_rows, int act, const float *filt_host,
                            const float *bias_host, pcnn_conv_plan **out) {
    PCNN_REQUIRE(ctx && filt_host && out, PCNN_ERR_ARG, "%s: NULL argument", fn);
    PCNN_REQUIRE_ACT(fn, act);
    ConvWideShape sh;
    int rc = conv_wide_shape(fn, N, H, W, C, K, R, S, stride, pad_h, pad_w, dil_h, dil_w, row_pitch, image_rows, &sh);
    if (rc) return rc;
    pcnn_device_guard g(ctx->device);
    std::unique_ptr<ConvWidePlan> pl(new ConvWidePlan());   // frees a half-built plan on every early return below
    pl->sh = sh;
    pl->N = N; pl->H = H; pl->W = W; pl->C = C; pl->row_pitch = row_pitch; pl->image_rows = image_rows > 0 ? image_rows : H;
    pl->act = act;
    ConvWideParams &p = pl->p;
    p.Pt = sh.Pt; p.Qt = sh.Qt; p.n_pb = sh.n_pb; p.n_qb = sh.n_qb; p.tiles = sh.tiles;
    p.R = R; p.S = S; p.stride = stride; p.nch = sh.nch; p.stages = sh.stages; p.K = K;
    p.taps = sh.taps;
    pl->cols = pl->pitch = R * S * C;
    pl->n = (long long)K * R * S * C;
    pl->K = K;
    if ((rc = pcnn_plan_upload(ctx, pl.get(), &pl->w, (size_t)pl->n * 2, filt_host, bias_host))) return rc;
    p.bias = pl->bias;
    {
        const uint64_t dims[3] = {(uint64_t)C, (uint64_t)R * S, (uint64_t)K};
        const uint64_t str[2] = {(uint64_t)C * 2, (uint64_t)R * S * C * 2};
        const uint32_t box[3] = {WD_KC, 1, (uint32_t)sh.npad};
        rc = make_map_bf16(&pl->map_w, pl->w, 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
        if (rc) return rc;
    }
    static bool configured[64] = {};        // function attributes are per device
    if (!configured[ctx->device & 63]) {
        for (int npad = 16; npad <= 256; npad += 16)
            for (int a : {PCNN_ACT_NONE, PCNN_ACT_SIGMOID, PCNN_ACT_RELU})
                PCNN_CUDA(cudaFuncSetAttribute(conv_wide_variant(a, npad), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               WD_SMEM_BUDGET + 2048));
        configured[ctx->device & 63] = true;
    }
    *out = pl.release();
    return PCNN_OK;
}

extern "C" int pcnn_conv_wide_plan_create(pcnn_ctx *ctx, int N, int H, int W, int C, int K, int R, int S, int stride, int row_pitch,
                                          int image_rows, int act, const float *filt_host, const float *bias_host,
                                          pcnn_conv_plan **out) {
    return wide_plan_create("pcnn_conv_wide_plan_create", ctx, N, H, W, C, K, R, S, stride, 0, 0, 1, 1, row_pitch, image_rows, act,
                            filt_host, bias_host, out);
}

extern "C" int pcnn_conv_wide_plan_create_padded(pcnn_ctx *ctx, int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h,
                                                 int pad_w, int row_pitch, int image_rows, int act, const float *filt_host,
                                                 const float *bias_host, pcnn_conv_plan **out) {
    return wide_plan_create("pcnn_conv_wide_plan_create_padded", ctx, N, H, W, C, K, R, S, stride, pad_h, pad_w, 1, 1, row_pitch,
                            image_rows, act, filt_host, bias_host, out);
}

extern "C" int pcnn_conv_wide_plan_create_dilated(pcnn_ctx *ctx, int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h,
                                                  int pad_w, int dil_h, int dil_w, int row_pitch, int image_rows, int act,
                                                  const float *filt_host, const float *bias_host, pcnn_conv_plan **out) {
    return wide_plan_create("pcnn_conv_wide_plan_create_dilated", ctx, N, H, W, C, K, R, S, stride, pad_h, pad_w, dil_h, dil_w, row_pitch,
                            image_rows, act, filt_host, bias_host, out);
}

int ConvWidePlan::fwd(pcnn_ctx *ctx, const void *x_bf16, void *y_bf16) {
    PCNN_REQUIRE(((uintptr_t)y_bf16 & 15) == 0, PCNN_ERR_ARG, "pcnn_conv_tc_fwd: the output must be 16-byte aligned (TMA stores)");
    ConvWideMaps m;
    memset(&m, 0, sizeof(m));
    m.w = map_w;
    int rc = conv_wide_x_maps(m.x, x_bf16, N, H, W, C, p.R, p.S, p.stride, sh.taps, row_pitch, image_rows, sh.Pt, sh.Qt);
    if (rc) return rc;
    {
        const uint64_t dims[4] = {(uint64_t)K, (uint64_t)sh.Q, (uint64_t)sh.P, (uint64_t)N};
        const uint64_t str[3] = {(uint64_t)K * 2, (uint64_t)sh.Q * K * 2, (uint64_t)sh.P * sh.Q * K * 2};
        const uint32_t box[4] = {64, (uint32_t)(sh.Pt >= 2 ? sh.Qt : 64), (uint32_t)(sh.Pt >= 2 ? sh.Pt / 2 : 1), 1};
        rc = make_map_bf16(&m.y, y_bf16, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE);
        if (rc) return rc;
    }
    const int grid = p.tiles < ctx->sm_count ? p.tiles : ctx->sm_count;
    void *args[] = {&m, &p};
    PCNN_CUDA(cudaLaunchKernel(conv_wide_variant(act, sh.npad), dim3((unsigned)grid), dim3(WD_THREADS), args,
                               wide_smem_bytes(sh.npad, p.stages), ctx->stream));
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
