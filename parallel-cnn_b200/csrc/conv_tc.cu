// parallel-cnn_b200/csrc/conv_tc.cu -- bf16 convolution forward on the Hopper tensor cores (SURVEY.md x3, BASELINE.json
// configs 3 and 5): wgmma with register accumulators, operands staged by TMA, no im2col pass.
//
// Formulation ("row-Toeplitz implicit GEMM").  The reference's conv is a valid, stride-1 cross-correlation
// (Sequential/layer.h:118-130); for NHWC activations one output row is
//     y[n][p][q][k] = sum_r  sum_{(w,c)}  x[n][p+r][w][c] * T_r[(w,c)][(q,k)],      T_r[(w,c)][(q,k)] = f[k][r][w-q][c]
// i.e. R GEMMs whose A operand is simply the input row p+r (W*C contiguous elements) and whose B operand is a banded
// Toeplitz matrix that depends only on (w - q).  Tiling the output row into blocks of Qt pixels makes the band a
// small CONSTANT matrix: for a block starting at q0 only the (Qt+S-1)*C <= 32 input elements from column q0*C matter,
// and T_r restricted to them is the same [32 x Qt*K] matrix for every block, every row and every image.  So
//   * A tiles are plain 2-D TMA boxes [128 rows x 32 elements] of the activation tensor viewed as [N*H][W*C]
//     (row r of the filter = the same box shifted down by r rows): zero im2col traffic, the 16x..25x expansion of
//     im2col never exists anywhere, not even in shared memory;
//   * B = R matrices [Qt*K x 32] (<= 48 KB) built once on the host from the filter bank, resident in shared memory;
//   * D = [128 x Qt*K] fp32 in the registers of two warpgroups (64 rows each, N = Qt*K rounded up to 32 <= 256);
//   * per tile and warpgroup 2*R wgmma (M=64, N, K=16), then the epilogue (bias, optional sigmoid, bf16 pack, store)
//     straight from the accumulator registers while the producer warp already stages the next tiles.
// Density: LeNet c1 (C=1, K=6, 5x5, Qt=24): 25/32 of K and 6*24/144 of N are useful but the band itself is sparse
// (17 % of the issued MACs are useful); config 5 (C=3, K=64, 3x3, Qt=4): 28 %.  The tensor pipe has > 10x headroom over
// the HBM time of these layers (AI 10-26 flop/B), which is the point: the layer is HBM-bound and the tensor cores are
// what lets a bf16 kernel reach the HBM roofline where the fp32 FMA pipe cannot (SURVEY.md 8d).
//
//
// Warp roles (288 threads, 1 CTA/SM, persistent over tiles): warps 0-7 = two consumer warpgroups (MMA + epilogue, output rows
// 0-63 and 64-127 of a tile), warp 8 = TMA producer.
#include "tc_common.cuh"

#include <vector>

using namespace pcnn_tc;

namespace {

constexpr int TC_THREADS = 288;
constexpr int TC_CONSUMER_WARPS = 8;
constexpr int TC_M = 128;          // output rows per tile (two warpgroups of 64)
constexpr int TC_KCHUNK = 32;      // bf16 elements per filter row r (64 B = one SWIZZLE_64B span)
constexpr int TC_MAX_STAGES = 4;
constexpr int TC_SMEM_BUDGET = 225 * 1024;
constexpr int TC_MAX_R = 5;
constexpr int A_TILE_BYTES = TC_M * TC_KCHUNK * 2;   // 8 KB

struct ConvTcParams {
    int n_img, H, P, Q, K, R;      // images, input rows per image, valid output rows/cols, filters, filter rows
    int Qt, ncols, npad;           // output pixels per tile, Qt * K, MMA width (ncols rounded up to 32)
    int C;                         // input channels (column offset of a tile = q0 * stride * C elements)
    int stride;                    // step of the window in both directions (1 = the reference's conv, layer.h:118-130)
    int x_pitch;                   // elements between input rows: filter row r of a stride-s conv reads view row r / s at
                                   // column offset (r % s) * x_pitch of the input viewed as [N * H / s][s * x_pitch]
    int V;                         // Toeplitz variants: the box start is rounded down to 8 elements (16 B, a TMA
                                   // requirement on the global address), the remainder (q0*C) % 8 selects the variant
    int stages;                    // activation stages that fit next to the V * R Toeplitz matrices
    int n_mtiles, n_qtiles;
    int act;                       // 0: none, 1: sigmoid (the reference's activation, layer.h:81-83)
    long long y_row_elems;         // Q * K
    __nv_bfloat16 *y;
    const float *bias;             // [K] or null
};

// dynamic shared memory, 1024-byte aligned:  [V*R Toeplitz matrices of npad*64 B] [stages*R activation tiles of 8 KB] [ctl]
struct ConvTcCtl {
    float bias[256];
    unsigned long long full[TC_MAX_STAGES], empty[TC_MAX_STAGES], bfull;
};
struct ConvTcSmemView {
    unsigned char *base;
    int R, bmat, stages, V;
    __device__ __forceinline__ unsigned char *b(int v, int r) const { return base + (size_t)(v * R + r) * bmat; }
    __device__ __forceinline__ unsigned char *a(int stage, int r) const {
        return base + (size_t)V * R * bmat + (size_t)(stage * R + r) * A_TILE_BYTES;
    }
    __device__ __forceinline__ ConvTcCtl &ctl() const {
        return *reinterpret_cast<ConvTcCtl *>(base + (size_t)V * R * bmat + (size_t)stages * R * A_TILE_BYTES);
    }
};
static size_t conv_tc_smem_bytes(int V, int R, int npad, int stages) {
    return (size_t)V * R * npad * TC_KCHUNK * 2 + (size_t)stages * R * A_TILE_BYTES + sizeof(ConvTcCtl) + 1024;
}

// sigmoid for a bf16 result: 0.5 + 0.5 tanh(x / 2) with ONE transcendental (MUFU.TANH) instead of two (EX2 + RCP).
// tanh.approx is good to ~5e-4 absolute, a quarter of a bf16 ulp of the result; the test bound (2^-8 |ref| + 1e-3) is unchanged.
__device__ __forceinline__ float sigmoid_bf16(float x) {
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * x));
    return fmaf(t, 0.5f, 0.5f);
}

// ACT (0 none, 1 sigmoid) and the MMA width N are compile-time; a missing bias reads as zeros from the shared bias table
template <int ACT, int N>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_conv_tc_fwd(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_b, const ConvTcParams p) {
    extern __shared__ unsigned char smem_dyn[];
    ConvTcSmemView sv;
    sv.base = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    sv.R = p.R; sv.bmat = N * TC_KCHUNK * 2; sv.stages = p.stages; sv.V = p.V;
    ConvTcCtl &S = sv.ctl();
    const int NST = p.stages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ntiles = p.n_mtiles * p.n_qtiles;

    if (threadIdx.x == 0) {
        for (int i = 0; i < NST; ++i) { bar_init(&S.full[i], 1); bar_init(&S.empty[i], TC_CONSUMER_WARPS); }
        bar_init(&S.bfull, 1);
        fence_barrier_init();
    }
    for (int i = threadIdx.x; i < 256; i += TC_THREADS) S.bias[i] = (p.bias && i < p.ncols) ? p.bias[i % p.K] : 0.0f;
    __syncthreads();

    if (warp == TC_CONSUMER_WARPS) {
        // ===== TMA producer: the Toeplitz operand once, then R activation boxes per tile =====
        if (lane == 0) {
            bar_expect_tx(&S.bfull, (unsigned)(p.V * p.R * N * TC_KCHUNK * 2));
            for (int v = 0; v < p.V; ++v)
                for (int r = 0; r < p.R; ++r) tma_load_2d(sv.b(v, r), &map_b, 0, (v * p.R + r) * N, &S.bfull);
            int it = 0;
            for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
                const int stage = it % NST;
                const unsigned ph = (unsigned)(it / NST) & 1u;
                bar_wait_relaxed(&S.empty[stage], ph ^ 1u, 32);
                const int mt = tile / p.n_qtiles, qt = tile % p.n_qtiles;
                bar_expect_tx(&S.full[stage], (unsigned)(p.R * A_TILE_BYTES));
                for (int r = 0; r < p.R; ++r)
                    tma_load_2d(sv.a(stage, r), &map_x, ((qt * p.Qt * p.stride * p.C) & ~7) + (r % p.stride) * p.x_pitch,
                                mt * TC_M + r / p.stride, &S.full[stage]);
            }
        }
        return;
    }

    // ===== consumer warpgroups: MMA into registers, then bias / activation -> bf16 -> HBM =====
    const int wg = warp >> 2, wq = warp & 3;
    const uint32_t bias_s = s_u32(S.bias);
    bar_wait(&S.bfull, 0);
    int it = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
        const int stage = it % NST;
        const unsigned ph = (unsigned)(it / NST) & 1u;
        const int mt = tile / p.n_qtiles, qt = tile % p.n_qtiles;
        const int var = qt % p.V;                          // which 16-byte remainder this pixel block starts at
        float acc[N / 2];
        bar_wait(&S.full[stage], ph);
        wg_fence();
        for (int r = 0; r < p.R; ++r) {
            const uint32_t a0 = s_u32(sv.a(stage, r)) + (uint32_t)(wg * 64 * TC_KCHUNK * 2), b0 = s_u32(sv.b(var, r));
#pragma unroll
            for (int ks = 0; ks < TC_KCHUNK / 16; ++ks)    // K = 16 bf16 = 32 bytes per instruction
                wgmma_bf16<0, 0>(acc, gmma_desc_k_sw64(a0 + ks * 32), gmma_desc_k_sw64(b0 + ks * 32), (r | ks) != 0 ? 1u : 0u);
        }
        wg_commit();
        wg_wait<0>();
        wg_hold(acc);
        __syncwarp();
        if (lane == 0) bar_arrive(&S.empty[stage]);       // smem stage reusable: this warp's MMAs have retired

        const int q0 = qt * p.Qt;
        int valid_cols = (p.Q - q0) * p.K;
        if (valid_cols > p.ncols) valid_cols = p.ncols;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const long long m = (long long)mt * TC_M + wg * 64 + wg_row(2 * h, wq, lane);   // output row n * H + p
            const int n = (int)(m / p.H), pr = (int)(m % p.H);
            if (n >= p.n_img || pr >= p.P) continue;
            __nv_bfloat16 *yrow = p.y + ((long long)n * p.P + pr) * p.y_row_elems + (long long)q0 * p.K;
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                const int c = wg_col(4 * j, lane);
                if (c >= valid_cols) continue;
                float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
                float2 bb;
                asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(bb.x), "=f"(bb.y) : "r"(bias_s + (uint32_t)c * 4u));
                f0 += bb.x; f1 += bb.y;
                if (ACT == 1) { f0 = sigmoid_bf16(f0); f1 = sigmoid_bf16(f1); }
                if (c + 1 < valid_cols && ((reinterpret_cast<uintptr_t>(yrow + c) & 3) == 0)) {
                    *reinterpret_cast<__nv_bfloat162 *>(yrow + c) = __floats2bfloat162_rn(f0, f1);
                } else {
                    yrow[c] = __float2bfloat16_rn(f0);
                    if (c + 1 < valid_cols) yrow[c + 1] = __float2bfloat16_rn(f1);
                }
            }
        }
    }
}

typedef void (*conv_tc_fwd_fn)(const CUtensorMap, const CUtensorMap, const ConvTcParams);
#define PCNN_FWD_ROW(N) {k_conv_tc_fwd<0, N>, k_conv_tc_fwd<1, N>}
static const void *conv_tc_fwd_variant(bool sigmoid, int npad) {
    static const conv_tc_fwd_fn table[8][2] = {PCNN_FWD_ROW(32),  PCNN_FWD_ROW(64),  PCNN_FWD_ROW(96),  PCNN_FWD_ROW(128),
                                               PCNN_FWD_ROW(160), PCNN_FWD_ROW(192), PCNN_FWD_ROW(224), PCNN_FWD_ROW(256)};
    return reinterpret_cast<const void *>(table[npad / 32 - 1][sigmoid ? 1 : 0]);
}
#undef PCNN_FWD_ROW


// fp32 [rows][w] -> bf16 [rows][pitch] (zero padded), for building the padded NHWC activations the TMA map needs
__global__ void k_f32_to_bf16_rows(const float *__restrict__ src, __nv_bfloat16 *__restrict__ dst, long rows, int w, int pitch) {
    const long total = rows * pitch;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const long r = i / pitch;
        const int c = (int)(i % pitch);
        dst[i] = __float2bfloat16_rn(c < w ? src[r * w + c] : 0.0f);
    }
}

int make_map_2d(CUtensorMap *map, void *base, uint64_t inner, uint64_t outer, uint64_t pitch_bytes, uint32_t box_inner, uint32_t box_outer) {
    encode_tiled_fn enc;
    int rc = get_encode(&enc);
    if (rc) return rc;
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {pitch_bytes};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        pcnn_set_error("cuTensorMapEncodeTiled failed (%d) for [%llu x %llu] pitch %llu box [%u x %u]", (int)r,
                       (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)pitch_bytes, box_inner, box_outer);
        return PCNN_ERR_CUDA;
    }
    return PCNN_OK;
}

}  // namespace

struct pcnn_conv_plan {
    ConvTcParams p;
    int W, S, row_pitch, stride, in_image_rows;
    void *d_toeplitz = nullptr;     // [R][ncols][32] bf16
    float *d_bias = nullptr;
    CUtensorMap map_b;
};

static void free_plan(pcnn_conv_plan *plan) {
    if (!plan) return;
    if (plan->d_toeplitz) cudaFree(plan->d_toeplitz);
    if (plan->d_bias) cudaFree(plan->d_bias);
    delete plan;
}

extern "C" int pcnn_conv_tc_plan_create(pcnn_ctx *ctx, int N, int H, int W, int C, int K, int R, int S, int row_pitch,
                                        int image_rows, int act, const float *filt_host, const float *bias_host,
                                        pcnn_conv_plan **out) {
    return pcnn_conv_tc_plan_create_strided(ctx, N, H, W, C, K, R, S, 1, row_pitch, image_rows, act, filt_host, bias_host, out);
}

extern "C" int pcnn_conv_tc_plan_create_strided(pcnn_ctx *ctx, int N, int H, int W, int C, int K, int R, int S, int stride, int row_pitch,
                                                int image_rows, int act, const float *filt_host, const float *bias_host,
                                                pcnn_conv_plan **out) {
    PCNN_REQUIRE(ctx && filt_host && out, PCNN_ERR_ARG, "pcnn_conv_tc_plan_create: NULL argument");
    PCNN_REQUIRE(stride >= 1 && stride <= 4, PCNN_ERR_ARG, "pcnn_conv_tc_plan_create: stride %d outside 1..4", stride);
    PCNN_REQUIRE(N > 0 && H >= R && W >= S && C > 0 && K > 0 && R > 0 && R <= TC_MAX_R && S > 0, PCNN_ERR_ARG,
                 "pcnn_conv_tc_plan_create: bad shape N=%d H=%d W=%d C=%d K=%d R=%d S=%d", N, H, W, C, K, R, S);
    PCNN_REQUIRE(row_pitch >= W * C && row_pitch % 8 == 0, PCNN_ERR_ARG,
                 "pcnn_conv_tc_plan_create: row pitch %d must be >= W*C and a multiple of 8 elements (TMA 16-byte strides)", row_pitch);
    if (image_rows <= 0) image_rows = H;
    PCNN_REQUIRE(image_rows >= H, PCNN_ERR_ARG, "pcnn_conv_tc_plan_create: image pitch of %d rows is smaller than H = %d", image_rows, H);
    PCNN_REQUIRE(image_rows % stride == 0, PCNN_ERR_ARG,
                 "pcnn_conv_tc_plan_create: rows per image (%d) must be a multiple of the stride %d (the input is addressed as [N * rows / stride] "
                 "rows of stride * pitch elements)", image_rows, stride);
    const int Q = (W - S) / stride + 1, P = (H - R) / stride + 1;
    // pixel block Qt: the TMA box must start on a 16-byte boundary, so it starts at (q0*C) & ~7 and the Toeplitz
    // operand absorbs the remainder delta = (q0*C) % 8: delta + (Qt+S-1)*C elements must fit the 32-element K chunk.
    // q0 = qt * Qt, so delta cycles with period V = 8 / gcd(8, Qt*C); each remainder needs its own operand copy.
    auto gcd = [](int a, int b) { while (b) { int t = a % b; a = b; b = t; } return a; };
    int Qt = 0, V = 1, stages = 0;
    for (int t = Q; t >= 1 && !Qt; --t) {
        if (t * K > 256 || (t * K) % 16 != 0) continue;
        const int single = ((Q + t - 1) / t) == 1;                       // one block per row: delta is always 0
        const int v = single ? 1 : 8 / gcd(8, (t * stride * C) % 8 == 0 ? 8 : (t * stride * C) % 8);
        int max_delta = 0;
        for (int i = 0; i < v; ++i) max_delta = max_delta > (i * t * stride * C) % 8 ? max_delta : (i * t * stride * C) % 8;
        if (max_delta + ((t - 1) * stride + S) * C > TC_KCHUNK) continue;
        const size_t fixed = (size_t)v * R * ((t * K + 31) / 32 * 32) * TC_KCHUNK * 2 + sizeof(ConvTcCtl) + 1024;
        if (fixed + 2 * (size_t)R * A_TILE_BYTES > (size_t)TC_SMEM_BUDGET) continue;
        int st = (int)(((size_t)TC_SMEM_BUDGET - fixed) / ((size_t)R * A_TILE_BYTES));
        Qt = t; V = v; stages = st > TC_MAX_STAGES ? TC_MAX_STAGES : st;
    }
    PCNN_REQUIRE(Qt > 0, PCNN_ERR_ARG,
                 "pcnn_conv_tc_plan_create: no pixel block with ((Qt-1)*stride+S)*C (+ alignment remainder) <= 32, Qt*K <= 256, %%16 == 0");
    pcnn_device_guard g(ctx->device);
    struct PlanGuard {                       // frees a half-built plan on every early return below
        pcnn_conv_plan *p;
        ~PlanGuard() { free_plan(p); }
    } guard{new pcnn_conv_plan()};
    pcnn_conv_plan *pl = guard.p;
    pl->W = W; pl->S = S; pl->row_pitch = row_pitch; pl->stride = stride; pl->in_image_rows = image_rows;
    ConvTcParams &p = pl->p;
    // rows are counted in units of `stride` input rows: tile row m = n * (image_rows / stride) + p
    p.n_img = N; p.H = image_rows / stride; p.P = P; p.Q = Q; p.K = K; p.R = R; p.Qt = Qt; p.ncols = Qt * K; p.npad = (Qt * K + 31) / 32 * 32; p.C = C; p.V = V; p.stages = stages;
    p.stride = stride; p.x_pitch = row_pitch;
    p.n_mtiles = (int)(((long long)N * p.H + TC_M - 1) / TC_M);
    p.n_qtiles = (Q + Qt - 1) / Qt;
    p.act = act;
    p.y_row_elems = (long long)Q * K;
    // Toeplitz operands: T_{v,r}[(ql, k)][kk] = f[k][r][s][c] where kk = delta_v + (ql + s) * C + c; rows ncols..npad-1 stay zero
    std::vector<uint16_t> t((size_t)V * R * p.npad * TC_KCHUNK, 0);
    for (int v = 0; v < V; ++v) {
        const int delta = (v * Qt * stride * C) % 8;
        for (int r = 0; r < R; ++r)
            for (int ql = 0; ql < Qt; ++ql)
                for (int k = 0; k < K; ++k)
                    for (int s = 0; s < S; ++s)
                        for (int c = 0; c < C; ++c)
                            t[(((size_t)v * R + r) * p.npad + ql * K + k) * TC_KCHUNK + delta + (ql * stride + s) * C + c] =
                                f32_to_bf16_bits(filt_host[(((size_t)k * R + r) * S + s) * C + c]);
    }
    PCNN_CUDA(cudaMalloc(&pl->d_toeplitz, t.size() * 2));
    PCNN_CUDA(cudaMemcpy(pl->d_toeplitz, t.data(), t.size() * 2, cudaMemcpyHostToDevice));
    if (bias_host) {
        PCNN_CUDA(cudaMalloc((void **)&pl->d_bias, K * sizeof(float)));
        PCNN_CUDA(cudaMemcpy(pl->d_bias, bias_host, K * sizeof(float), cudaMemcpyHostToDevice));
    }
    p.bias = pl->d_bias;
    int rc = make_map_2d(&pl->map_b, pl->d_toeplitz, TC_KCHUNK, (uint64_t)V * R * p.npad, TC_KCHUNK * 2, TC_KCHUNK, (uint32_t)p.npad);
    if (rc) return rc;
    static bool configured[64] = {};        // function attributes are per device
    if (!configured[ctx->device & 63]) {
        for (int v = 0; v < 16; ++v)
            PCNN_CUDA(cudaFuncSetAttribute(conv_tc_fwd_variant(v & 1, 32 * (v / 2 + 1)), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           TC_SMEM_BUDGET + 2048));
        configured[ctx->device & 63] = true;
    }
    guard.p = nullptr;
    *out = pl;
    return PCNN_OK;
}

extern "C" int pcnn_conv_tc_plan_destroy(pcnn_ctx *ctx, pcnn_conv_plan *plan) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_conv_tc_plan_destroy: ctx is NULL");
    if (!plan) return PCNN_OK;
    pcnn_device_guard g(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    free_plan(plan);
    return PCNN_OK;
}

extern "C" int pcnn_conv_tc_fwd(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *x_bf16, void *y_bf16) {
    PCNN_REQUIRE(ctx && plan && x_bf16 && y_bf16, PCNN_ERR_ARG, "pcnn_conv_tc_fwd: NULL argument");
    PCNN_REQUIRE(((uintptr_t)x_bf16 & 15) == 0, PCNN_ERR_ARG, "pcnn_conv_tc_fwd: activations must be 16-byte aligned");
    pcnn_device_guard g(ctx->device);
    ConvTcParams p = plan->p;
    p.y = reinterpret_cast<__nv_bfloat16 *>(y_bf16);
    CUtensorMap map_x;
    // stride s: the input viewed as [N * rows / s] rows of s * pitch elements (see ConvTcParams::x_pitch)
    int rc = make_map_2d(&map_x, const_cast<void *>(x_bf16), (uint64_t)plan->row_pitch * plan->stride, (uint64_t)p.n_img * p.H,
                         (uint64_t)plan->row_pitch * plan->stride * 2, TC_KCHUNK, TC_M);
    if (rc) return rc;
    const int ntiles = p.n_mtiles * p.n_qtiles;
    const int grid = ntiles < ctx->sm_count ? ntiles : ctx->sm_count;
    void *args[] = {&map_x, &plan->map_b, &p};
    PCNN_CUDA(cudaLaunchKernel(conv_tc_fwd_variant(p.act == 1, p.npad), dim3((unsigned)grid), dim3(TC_THREADS), args,
                               conv_tc_smem_bytes(p.V, p.R, p.npad, p.stages), ctx->stream));
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_f32_to_bf16_rows(pcnn_ctx *ctx, const float *src, void *dst_bf16, long rows, int w, int pitch) {
    PCNN_REQUIRE(ctx && src && dst_bf16 && rows > 0 && w > 0 && pitch >= w, PCNN_ERR_ARG, "pcnn_f32_to_bf16_rows: bad argument");
    pcnn_device_guard g(ctx->device);
    long blocks = (rows * pitch + 255) / 256;
    if (blocks > (long)ctx->sm_count * 16) blocks = (long)ctx->sm_count * 16;
    k_f32_to_bf16_rows<<<(int)blocks, 256, 0, ctx->stream>>>(src, reinterpret_cast<__nv_bfloat16 *>(dst_bf16), rows, w, pitch);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
