// parallel-cnn_b200/csrc/diag_kernels.cu -- measurement helper: how fast can one SM-resident TMA pipeline stream a bf16 tensor
// [N][P][Q][64] out of HBM with the box shapes the convolution kernels use?  The kernel is the load pipeline of
// the convolution backward kernels with the tensor-core work removed (the consumer releases every stage as soon as it lands), so its rate
// is the ceiling those kernels can reach with that access pattern; bench scripts print it next to the kernels' own rate.
#include "tc_common.cuh"

using namespace pcnn_tc;

namespace {

constexpr int DS_MAX_STAGES = 12;
constexpr int DS_SMEM = 200 * 1024;

struct StreamParams {
    int mode, stages, stage_bytes;
    int N, P, Q;
    long long nchunks;
    const unsigned char *base;
};

struct StreamCtl {
    unsigned long long full[DS_MAX_STAGES], empty[DS_MAX_STAGES];
};

// mode 0: 1-D bulk copies of 16 KB        mode 1: 2-D boxes {64 ch, 128 pixels} (16 KB contiguous, 128-byte rows, swizzled)
// mode 2: dgrad pattern, 4 boxes {64 ch, 1 pixel, 32 rows} per 16 KB stage   mode 3: wgrad pattern, one box {64 ch, Qpad pixels, 1 row}
__global__ void __launch_bounds__(64, 1)
k_tma_stream(const __grid_constant__ CUtensorMap map, const StreamParams p, unsigned *sink) {
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *base = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    StreamCtl &S = *reinterpret_cast<StreamCtl *>(base + (size_t)p.stages * p.stage_bytes);
    const int NST = p.stages;
    if (threadIdx.x == 0) {
        for (int i = 0; i < NST; ++i) { bar_init(&S.full[i], 1); bar_init(&S.empty[i], 1); }
        fence_barrier_init();
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        int it = 0;
        for (long long ch = blockIdx.x; ch < p.nchunks; ch += gridDim.x, ++it) {
            const int stage = it % NST;
            const unsigned ph = (unsigned)(it / NST) & 1u;
            bar_wait(&S.empty[stage], ph ^ 1u);
            unsigned char *dst = base + (size_t)stage * p.stage_bytes;
            bar_expect_tx(&S.full[stage], (unsigned)p.stage_bytes);
            if (p.mode == 0) {
                tma_load_1d(dst, p.base + ch * p.stage_bytes, (unsigned)p.stage_bytes, &S.full[stage]);
            } else if (p.mode == 1) {
                tma_load_2d(dst, &map, 0, (int)(ch * 128), &S.full[stage]);
            } else if (p.mode == 2) {
                const int q = (int)(ch % p.Q), hb = (int)((ch / p.Q) % 2), n = (int)(ch / (2LL * p.Q));
                for (int g = 0; g < 4; ++g) tma_load_4d(dst + g * 4096, &map, 0, q, hb * 120 + g * 30 - 2, n, &S.full[stage]);
            } else {
                tma_load_3d(dst, &map, 0, 0, (int)ch, &S.full[stage]);
            }
        }
    } else if (warp == 1 && lane == 0) {
        int it = 0;
        unsigned acc = 0;
        for (long long ch = blockIdx.x; ch < p.nchunks; ch += gridDim.x, ++it) {
            const int stage = it % NST;
            const unsigned ph = (unsigned)(it / NST) & 1u;
            bar_wait(&S.full[stage], ph);
            acc += *reinterpret_cast<volatile unsigned *>(base + (size_t)stage * p.stage_bytes);
            bar_arrive(&S.empty[stage]);
        }
        if (acc == 0x12345678u) *sink = acc;
    }
}

}  // namespace

extern "C" int pcnn_measure_tma_read(pcnn_ctx *ctx, const void *dev_bf16, int N, int P, int Q, int mode, int iters, float *gbps_out) {
    PCNN_REQUIRE(ctx && dev_bf16 && gbps_out && N > 0 && P > 0 && Q > 0 && mode >= 0 && mode <= 3 && iters > 0, PCNN_ERR_ARG,
                 "pcnn_measure_tma_read: bad argument");
    PCNN_REQUIRE(((uintptr_t)dev_bf16 & 15) == 0, PCNN_ERR_ARG, "pcnn_measure_tma_read: tensor must be 16-byte aligned");
    pcnn_device_guard g(ctx->device);
    StreamParams p;
    memset(&p, 0, sizeof(p));
    p.mode = mode; p.N = N; p.P = P; p.Q = Q;
    p.base = reinterpret_cast<const unsigned char *>(dev_bf16);
    const long long pixels = (long long)N * P * Q;
    CUtensorMap map;
    memset(&map, 0, sizeof(map));
    int rc = PCNN_OK;
    if (mode == 0) {
        p.stage_bytes = 16384;
        p.nchunks = pixels * 128 / 16384;
    } else if (mode == 1) {
        p.stage_bytes = 16384;
        p.nchunks = pixels / 128;
        const uint64_t dims[2] = {64, (uint64_t)pixels};
        const uint64_t str[1] = {128};
        const uint32_t box[2] = {64, 128};
        rc = make_map_bf16(&map, const_cast<void *>(dev_bf16), 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    } else if (mode == 2) {
        PCNN_REQUIRE(P <= 238, PCNN_ERR_ARG, "pcnn_measure_tma_read: mode 2 walks two row blocks of 120 per image");
        p.stage_bytes = 16384;
        p.nchunks = (long long)N * 2 * Q;
        const uint64_t dims[4] = {64, (uint64_t)Q, (uint64_t)P, (uint64_t)N};
        const uint64_t str[3] = {128, (uint64_t)Q * 128, (uint64_t)P * Q * 128};
        const uint32_t box[4] = {64, 1, 32, 1};
        rc = make_map_bf16(&map, const_cast<void *>(dev_bf16), 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    } else {
        const int Qpad = (Q + 15) / 16 * 16;
        PCNN_REQUIRE(Qpad <= 256, PCNN_ERR_ARG, "pcnn_measure_tma_read: mode 3 needs Q <= 256");
        p.stage_bytes = Qpad * 128;
        p.nchunks = (long long)N * P;
        const uint64_t dims[3] = {64, (uint64_t)Q, (uint64_t)N * P};
        const uint64_t str[2] = {128, (uint64_t)Q * 128};
        const uint32_t box[3] = {64, (uint32_t)Qpad, 1};
        rc = make_map_bf16(&map, const_cast<void *>(dev_bf16), 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    }
    if (rc) return rc;
    p.stages = (int)((DS_SMEM - sizeof(StreamCtl) - 1024) / p.stage_bytes);
    if (p.stages > DS_MAX_STAGES) p.stages = DS_MAX_STAGES;
    const char *st = getenv("PCNN_DIAG_STAGES");
    if (st && atoi(st) > 0 && atoi(st) < p.stages) p.stages = atoi(st);
    static bool configured[64] = {};        // function attributes are per device
    if (!configured[ctx->device & 63]) {
        PCNN_CUDA(cudaFuncSetAttribute(k_tma_stream, cudaFuncAttributeMaxDynamicSharedMemorySize, DS_SMEM + 2048));
        configured[ctx->device & 63] = true;
    }
    const size_t smem = (size_t)p.stages * p.stage_bytes + sizeof(StreamCtl) + 1024;
    unsigned *sink = nullptr;
    if ((rc = pcnn_scratch(ctx, 64, (void **)&sink))) return rc;
    struct Events {                          // destroyed on every return path
        cudaEvent_t a = nullptr, b = nullptr;
        ~Events() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
    } ev;
    PCNN_CUDA(cudaEventCreate(&ev.a));
    PCNN_CUDA(cudaEventCreate(&ev.b));
    cudaEvent_t e0 = ev.a, e1 = ev.b;
    const int grid = p.nchunks < ctx->sm_count ? (int)p.nchunks : ctx->sm_count;
    for (int i = 0; i < 2; ++i) {
        k_tma_stream<<<grid, 64, smem, ctx->stream>>>(map, p, sink);
        PCNN_CHECK_LAUNCH(ctx);
    }
    PCNN_CUDA(cudaEventRecord(e0, ctx->stream));
    for (int i = 0; i < iters; ++i) {
        k_tma_stream<<<grid, 64, smem, ctx->stream>>>(map, p, sink);
        PCNN_CHECK_LAUNCH(ctx);
    }
    PCNN_CUDA(cudaEventRecord(e1, ctx->stream));
    PCNN_CUDA(cudaEventSynchronize(e1));
    float ms = 0.0f;
    PCNN_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    const double bytes = mode <= 1 ? (double)p.nchunks * p.stage_bytes : (double)pixels * 128.0;   // every byte of the tensor once
    *gbps_out = (float)(bytes * iters / (ms * 1e-3) / 1e9);
    return PCNN_OK;
}

namespace {

// ---- TMA store probe --------------------------------------------------------------------------------------------------
// How fast can the store half of the convolution forward epilogue run with everything else removed?  Output y viewed as
// [N][P][row_elems] bf16 (the forward kernel's own view); the grid walks tiles of 128 rows x 256 columns exactly like the
// forward kernel and every epilogue warp issues the stores of its rows from a (never written) shared-memory staging buffer:
//   mode 0: the forward kernel's pattern: 8 warps x 2 boxes {64 cols, 32 rows, 1 image}, SWIZZLE_128B (4 KB per instruction)
//   mode 1: 4 warps x 2 boxes {128 cols, 32 rows}, SWIZZLE_NONE (8 KB per instruction, 256-byte rows)
//   mode 2: 4 warps x 1 box {256 cols, 32 rows}, SWIZZLE_NONE (16 KB per instruction, 512-byte rows)
//   mode 3: mode 0 with every lane issuing 1-D bulk stores of its own 128-byte row piece (no tensor map)
//   mode 4: 4 warps x 4 boxes {64 cols, 32 rows} issued back to back by one lane, then one commit (group of 16 KB)
//   mode 5: no TMA: every lane writes its row's 128-byte piece with eight 16-byte st.global.v4 (STG.128, the widest on sm_90), 8 warps
//   mode 6: half and half: the even column boxes by TMA (mode 0), the odd ones by direct 16-byte stores (mode 5)
// `hot` = 1 makes every tile land on the first row block (an L2-resident target instead of HBM).
struct StoreParams {
    int mode, hot, n_img, P, H, n_mtiles, n_qtiles, row_elems;
    unsigned char *y;
};

__global__ void __launch_bounds__(256, 1) k_tma_store_probe(const __grid_constant__ CUtensorMap map, const StoreParams p) {
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *base = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ntiles = p.n_mtiles * p.n_qtiles;
    const int quarter = warp & 3, colhalf = warp >> 2;
    // modes 0, 1, 3: 2 x (4 or 8) KB per warp; modes 2, 4: 2 x 16 KB for each of the four issuing warps (128 KB in all)
    unsigned char *obuf = base + (size_t)warp * (p.mode == 2 || p.mode == 4 ? 32768 : 16384);
    int ob = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int mt = tile / p.n_qtiles, qt = tile % p.n_qtiles;
        const long long m0 = (long long)mt * 128 + quarter * 32;
        int n = (int)(m0 / p.H), pr = (int)(m0 % p.H);
        const bool ok = n < p.n_img && pr < p.P;
        if (p.hot) { n = 0; pr = pr % 32; }
        const int c_tile = qt * 256;
        if (p.mode == 5 || (p.mode == 6 && colhalf == 1)) {
            // direct path: every lane owns a row and writes its 128-byte piece as eight 16-byte stores from registers
            if (ok && pr + lane < p.P)
                for (int col0 = colhalf * 64; col0 < 256; col0 += 128) {
                    if (c_tile + col0 + 64 > p.row_elems) continue;
                    unsigned char *dst = p.y + (((long long)n * p.P + pr + lane) * p.row_elems + c_tile + col0) * 2;
#pragma unroll
                    for (int k = 0; k < 8; ++k)
                        asm volatile("st.global.v4.b32 [%0], {%1, %1, %1, %1};" ::"l"(dst + k * 16), "r"(tile + k / 2) : "memory");
                }
        } else if (p.mode == 0 || p.mode == 3 || p.mode == 6) {
            for (int col0 = colhalf * 64; col0 < 256; col0 += 128) {
                const uint32_t buf = s_u32(obuf + ob * 4096);
                if (p.mode != 3) {
                    if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                    __syncwarp();
                    if (lane == 0 && ok) {
                        asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(&map),
                                     "r"(c_tile + col0), "r"(pr), "r"(n), "r"(buf) : "memory");
                        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    }
                } else {
                    asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                    if (ok && pr + lane < p.P && c_tile + col0 + 64 <= p.row_elems) {
                        unsigned char *dst = p.y + (((long long)n * p.P + pr + lane) * p.row_elems + c_tile + col0) * 2;
                        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], 128;" ::"l"(dst), "r"(buf + lane * 128) : "memory");
                    }
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
                ob ^= 1;
            }
        } else if (p.mode == 1) {
            if (colhalf == 0)
                for (int col0 = 0; col0 < 256; col0 += 128) {
                    const uint32_t buf = s_u32(obuf + ob * 8192);
                    if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                    __syncwarp();
                    if (lane == 0 && ok) {
                        asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(&map),
                                     "r"(c_tile + col0), "r"(pr), "r"(n), "r"(buf) : "memory");
                        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    }
                    ob ^= 1;
                }
        } else if (p.mode == 2) {
            if (colhalf == 0) {
                const uint32_t buf = s_u32(obuf + ob * 16384);
                if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                __syncwarp();
                if (lane == 0 && ok) {
                    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(&map),
                                 "r"(c_tile), "r"(pr), "r"(n), "r"(buf) : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
                ob ^= 1;
            }
        } else {
            if (colhalf == 0) {
                const uint32_t buf = s_u32(obuf + ob * 16384);
                if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                __syncwarp();
                if (lane == 0 && ok) {
                    for (int b = 0; b < 4; ++b)
                        asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(&map),
                                     "r"(c_tile + b * 64), "r"(pr), "r"(n), "r"(buf + b * 4096) : "memory");
                    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                }
                ob ^= 1;
            }
        }
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

}  // namespace

extern "C" int pcnn_measure_tma_write(pcnn_ctx *ctx, void *dev_bf16, int N, int P, int H, int row_elems, int mode, int hot, int iters,
                                      float *gbps_out) {
    PCNN_REQUIRE(ctx && dev_bf16 && gbps_out && N > 0 && P > 0 && H >= P && H % 32 == 0 && row_elems > 0 && row_elems % 8 == 0 && mode >= 0 &&
                     mode <= 6 && iters > 0,
                 PCNN_ERR_ARG, "pcnn_measure_tma_write: bad argument");
    PCNN_REQUIRE(((uintptr_t)dev_bf16 & 15) == 0, PCNN_ERR_ARG, "pcnn_measure_tma_write: tensor must be 16-byte aligned");
    pcnn_device_guard g(ctx->device);
    StoreParams p;
    memset(&p, 0, sizeof(p));
    p.mode = mode; p.hot = hot; p.n_img = N; p.P = P; p.H = H; p.row_elems = row_elems;
    p.n_mtiles = (int)(((long long)N * H + 127) / 128);
    p.n_qtiles = (row_elems + 255) / 256;
    p.y = reinterpret_cast<unsigned char *>(dev_bf16);
    CUtensorMap map;
    memset(&map, 0, sizeof(map));
    const uint64_t dims[3] = {(uint64_t)row_elems, (uint64_t)P, (uint64_t)N};
    const uint64_t str[2] = {(uint64_t)row_elems * 2, (uint64_t)row_elems * 2 * P};
    const uint32_t cols = mode == 1 ? 128 : (mode == 2 ? 256 : 64);
    const uint32_t box[3] = {cols, 32, 1};
    int rc = make_map_bf16(&map, dev_bf16, 3, dims, str, box, cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                           CU_TENSOR_MAP_L2_PROMOTION_NONE);
    if (rc) return rc;
    const size_t smem = 128 * 1024 + 1024;
    static bool configured[64] = {};
    if (!configured[ctx->device & 63]) {
        PCNN_CUDA(cudaFuncSetAttribute(k_tma_store_probe, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured[ctx->device & 63] = true;
    }
    struct Events {
        cudaEvent_t a = nullptr, b = nullptr;
        ~Events() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
    } ev;
    PCNN_CUDA(cudaEventCreate(&ev.a));
    PCNN_CUDA(cudaEventCreate(&ev.b));
    const int ntiles = p.n_mtiles * p.n_qtiles;
    const int grid = ntiles < ctx->sm_count ? ntiles : ctx->sm_count;
    for (int i = 0; i < 2; ++i) {
        k_tma_store_probe<<<grid, 256, smem, ctx->stream>>>(map, p);
        PCNN_CHECK_LAUNCH(ctx);
    }
    PCNN_CUDA(cudaEventRecord(ev.a, ctx->stream));
    for (int i = 0; i < iters; ++i) {
        k_tma_store_probe<<<grid, 256, smem, ctx->stream>>>(map, p);
        PCNN_CHECK_LAUNCH(ctx);
    }
    PCNN_CUDA(cudaEventRecord(ev.b, ctx->stream));
    PCNN_CUDA(cudaEventSynchronize(ev.b));
    float ms = 0.0f;
    PCNN_CUDA(cudaEventElapsedTime(&ms, ev.a, ev.b));
    const double bytes = (double)N * P * row_elems * 2.0;        // the bytes of y (every one written once per launch when hot == 0)
    *gbps_out = (float)(bytes * iters / (ms * 1e-3) / 1e9);
    return PCNN_OK;
}

// ---- wgmma issue/throughput probe -------------------------------------------------------------------------------------
// One CTA of M / 64 warpgroups, each issuing `reps` back-to-back wgmma m64nNk16 on zero operands into its own register
// accumulator (the 64-row halves of an M = 128 product are independent, as in the forward kernel's two consumer
// warpgroups), then one wait; reports SM clocks per M x N x 16 product.  The convolution kernels size their MMAs against
// this table.
namespace {

// A_MN / B_MN: operand majors as compile-time constants, so the timed loop is one straight wgmma stream
template <int N, int A_MN, int B_MN>
__global__ void __launch_bounds__(256, 1) k_mma_rate(int reps, int walk, long long *out) {
    constexpr bool a_mn = A_MN != 0, b_mn = B_MN != 0;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *base = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    for (int i = threadIdx.x * 16; i < 96 * 1024; i += blockDim.x * 16) *reinterpret_cast<uint4 *>(base + i) = make_uint4(0, 0, 0, 0);
    fence_proxy_async_smem();
    const uint64_t ad = a_mn ? gmma_desc_mn_sw128(s_u32(base), 8192) : gmma_desc_k_sw128(s_u32(base));
    const uint64_t bd = b_mn ? gmma_desc_mn_sw128(s_u32(base + 32768), 8192) : gmma_desc_k_sw128(s_u32(base + 32768));
    // walk = 1: every MMA reads fresh operand tiles (A advances by its K-step footprint, B likewise, wrapping in 32 KB)
    const uint32_t a_adv = walk ? (uint32_t)((a_mn ? 2048 : 32) >> 4) : 0u, b_adv = walk ? (uint32_t)((b_mn ? 2048 : 32) >> 4) : 0u;
    const uint32_t a_wrap = a_mn ? 16u : 4u, b_wrap = b_mn ? 16u : 4u;     // steps before returning to the start
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.0f;
    wg_hold(acc);                                       // the zeroing stays ahead of the fence: one unbroken wgmma stream
    __syncthreads();
    const long long t0 = clock64();
    wg_fence();
    for (int i = 0; i < reps; ++i) {
        const uint64_t a = ad + (uint64_t)(((uint32_t)i % a_wrap) * a_adv), b = bd + (uint64_t)(((uint32_t)i % b_wrap) * b_adv);
        wgmma_bf16<A_MN, B_MN>(acc, a, b, 1u);
    }
    wg_commit();
    wg_wait<0>();
    wg_hold(acc);
    __syncthreads();
    const long long t1 = clock64();
    float s = 0.0f;
#pragma unroll
    for (int i = 0; i < N / 2; ++i) s += acc[i];
    if (threadIdx.x == 0) out[0] = t1 - t0 + (s != 0.0f ? 1 : 0);   // the operands are zero: s == 0 keeps the sum live only
}

typedef void (*mma_rate_fn)(int, int, long long *);
template <int... Ns> struct MmaRateTable {
    static const void *get(int N, int a_mn, int b_mn) {
        static const mma_rate_fn t[][4] = {{k_mma_rate<Ns, 0, 0>, k_mma_rate<Ns, 0, 1>, k_mma_rate<Ns, 1, 0>, k_mma_rate<Ns, 1, 1>}...};
        return reinterpret_cast<const void *>(t[N / 16 - 1][(a_mn ? 2 : 0) | (b_mn ? 1 : 0)]);
    }
};
using MmaRate = MmaRateTable<16, 32, 48, 64, 80, 96, 112, 128, 144, 160, 176, 192, 208, 224, 240, 256>;

}  // namespace

extern "C" int pcnn_measure_mma_rate(pcnn_ctx *ctx, int M, int N, int a_mn_major, int b_mn_major, int nacc, int reps, float *clk_per_mma) {
    PCNN_REQUIRE(ctx && clk_per_mma && (M == 64 || M == 128) && N >= 16 && N <= 256 && N % 16 == 0 && reps > 0 &&
                     (nacc == 1 || nacc == 2 || nacc == 4 || nacc == 8) && N * nacc <= 512,
                 PCNN_ERR_ARG, "pcnn_measure_mma_rate: bad argument");
    pcnn_device_guard g(ctx->device);
    const void *fn = MmaRate::get(N, a_mn_major, b_mn_major);
    static bool configured[64] = {};        // function attributes are per device
    if (!configured[ctx->device & 63]) {
        for (int n = 16; n <= 256; n += 16)
            for (int v = 0; v < 4; ++v)
                PCNN_CUDA(cudaFuncSetAttribute(MmaRate::get(n, v & 2, v & 1), cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        configured[ctx->device & 63] = true;
    }
    long long *out = nullptr;
    int rc = pcnn_scratch(ctx, 64, (void **)&out);
    if (rc) return rc;
    long long h = 0;
    for (int i = 0; i < 2; ++i) {      // second launch is the measurement (first warms the instruction cache)
        int walk = getenv("PCNN_MMA_WALK") ? atoi(getenv("PCNN_MMA_WALK")) : 1;
        void *args[] = {&reps, &walk, &out};
        PCNN_CUDA(cudaLaunchKernel(fn, dim3(1), dim3(128 * (M / 64)), args, 98 * 1024, ctx->stream));
        PCNN_CHECK_LAUNCH(ctx);
    }
    PCNN_CUDA(cudaMemcpyAsync(&h, out, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    *clk_per_mma = (float)h / (float)reps;
    return PCNN_OK;
}
