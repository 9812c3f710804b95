// parallel-cnn_b200/csrc/fused_body.cuh -- device code shared by the fused kernels: the per-image forward/backward
// pass of one CTA and the CTA-level reduction of its register accumulators.  See fused_kernels.cu for the design notes.
#pragma once
#include "pcnn_internal.h"

namespace pcnn_fused {

constexpr int NT = FUSED_THREADS;
constexpr int NWK = FUSED_WORKERS;
constexpr int NWARP = NT / 32;          // 7
constexpr int RED_STRIDE = 27;          // 25 c1 taps + c1 bias sum, padded to an odd stride

// the buffers of one image stream through 224 threads: staging, fp32 image, per-image reduction scratch
template <typename InT> struct ImageSmem {
    alignas(16) float imgf[2][PCNN_IMG];             // fp32 image, double buffered
    alignas(16) InT stage[2][PCNN_IMG];              // raw staging target of the bulk copies (u8 path only)
    alignas(16) float red[NWK * RED_STRIDE];         // epilogue scratch
    float fc_red[NWARP][PCNN_F];
    float red_s1[NWARP][17];
    int label[2];
    alignas(8) unsigned long long mbar[2];           // image stages
};

// what half 1 of a two-image CTA (persistent kernel) hands to half 0, which adds it to its own image's entries (image 0 +
// image 1) and pushes each packed entry once
struct PairXchg {
    float fw[PCNN_F][NWK];                           // f-layer weight gradient, column t of worker t
    float fb[PCNN_F + 1];                            // f bias gradient, error
    float tail[173];                                 // c1 taps + c1 bias sums (36 windows), s1 taps + s1 bias (7 warps)
};

template <typename InT> struct FusedSmem : ImageSmem<InT> {
    alignas(16) float params[NPACK];                 // packed parameters (9,376 B)
    float dpre_f[PCNN_F];
    float f_out[PCNN_F];
    float part[NT];                                  // persistent kernel: slot-phase partial sums of the owned chunk
    alignas(16) float recv[NPACK + 16];              // persistent kernel: [cluster rank][my share] gradient pieces pushed by the peers
    float accf[PCNN_F * NT];                         // persistent kernel, several images per CTA: thread-private sums of the f-layer weight gradient
    float lut[256];                                  // u8 pixel -> fp32 (mnist.h:145 + Main.cpp:64), filled once per kernel
    alignas(8) unsigned long long params_bar;        // parameters (bulk copy or peer pushes)
    alignas(8) unsigned long long grads_bar;         // gradient pieces pushed by the cluster peers
    // host-streaming gate of the persistent kernel (written and read by thread 0 only)
    const void *gate_images;
    const unsigned *gate_ready;
    pcnn_chunking gate_chunks;
    int *gate_abort;
    unsigned gate_tag;
    int aborted;                                     // persistent kernel: a wait of this CTA has given up; later waits return at once
};

// ---- mbarrier / bulk-copy helpers (PTX ISA: mbarrier, cp.async.bulk) -------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, unsigned bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// ---- flag-in-data words: {fp32 value (low half), tag (high half)} in ONE naturally aligned 64-bit scalar access, which
// the PTX memory model makes single-copy atomic.  The consumer polls the word itself until the tag matches, so neither
// side needs a fence or a separate flag round trip (the idea of NCCL's LL protocol, applied to L2-resident buffers).
typedef unsigned long long llword;
__device__ __forceinline__ void ll_store(llword *p, float v, unsigned tag) {
    asm volatile("{ .reg .b64 t; mov.b64 t, {%1, %2}; st.relaxed.gpu.global.u64 [%0], t; }" ::"l"(p), "r"(__float_as_uint(v)),
                 "r"(tag)
                 : "memory");
}
__device__ __forceinline__ void ll_load(const llword *p, float &v, unsigned &tag) {
    unsigned lo;
    asm volatile("{ .reg .b64 t; ld.relaxed.gpu.global.u64 t, [%2]; mov.b64 {%0, %1}, t; }" : "=r"(lo), "=r"(tag) : "l"(p) : "memory");
    v = __uint_as_float(lo);
}
// two consecutive words (16-byte aligned): two independent 64-bit accesses as far as atomicity goes
__device__ __forceinline__ void ll_load2(const llword *p, float &v0, unsigned &tag0, float &v1, unsigned &tag1) {
    unsigned a, b;
    asm volatile("{ .reg .b64 t, u; ld.relaxed.gpu.global.v2.u64 {t, u}, [%4]; mov.b64 {%0, %1}, t; mov.b64 {%2, %3}, u; }"
                 : "=r"(a), "=r"(tag0), "=r"(b), "=r"(tag1)
                 : "l"(p)
                 : "memory");
    v0 = __uint_as_float(a);
    v1 = __uint_as_float(b);
}

// ---- thread-block clusters: ranks, the hardware cluster barrier, distributed shared memory ----------------------------
__device__ __forceinline__ unsigned cluster_ctarank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ unsigned cluster_nctarank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ unsigned cluster_idx() {
    unsigned r;
    asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
    return r;
}
// all threads of all CTAs of the cluster; release/acquire also orders the distributed-shared-memory accesses around it
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t dsmem_addr(const void *own_smem, unsigned rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(own_smem)), "r"(rank));
    return r;
}
__device__ __forceinline__ void dsmem_st_f2(uint32_t addr, float x, float y) {
    asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(x), "f"(y) : "memory");
}
// asynchronous store into (any) CTA of the cluster that signals the destination CTA's mbarrier with its byte count: the
// receiver needs no barrier and no fence, it waits on its own mbarrier like for a bulk copy
__device__ __forceinline__ void dsmem_st_async_f32(uint32_t addr, float v, uint32_t mbar_addr) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.f32 [%0], %1, [%2];" ::"r"(addr), "f"(v), "r"(mbar_addr)
                 : "memory");
}
__device__ __forceinline__ void dsmem_st_async_f2(uint32_t addr, float x, float y, uint32_t mbar_addr) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];" ::"r"(addr), "f"(x), "f"(y),
                 "r"(mbar_addr)
                 : "memory");
}
// named CTA barrier as a one-way hand-over: the producers' arrive (no wait) releases their shared-memory stores to the
// consumers' sync; `n` counts the threads of both sides
__device__ __forceinline__ void named_bar_arrive(unsigned bar, unsigned n) {
    asm volatile("bar.arrive %0, %1;" ::"r"(bar), "r"(n) : "memory");
}
__device__ __forceinline__ void named_bar_sync(unsigned bar, unsigned n) {
    asm volatile("bar.sync %0, %1;" ::"r"(bar), "r"(n) : "memory");
}
__device__ __forceinline__ float dsmem_ld_f(uint32_t addr) {
    float v;
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
    return v;
}

// 1 / (1 + e^-v) = 1 / (1 + 2^(-v log2 e)): MUFU.EX2 + MUFU.RCP.  The exponent product is rounded to fp32, so the
// relative error of e^-v grows like |v| * 6e-8 (|v| < 30 here); the sigmoid inherits at most (1 - sigma) of it.
__device__ __forceinline__ float sigmoid_fast(float v) {
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * -1.4426950408889634f));
    return __fdividef(1.0f, 1.0f + e);
}

__device__ __forceinline__ float warp_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}


// Sixteen sums over the warp at once, "transposed": every round halves the number of values a lane holds instead of the
// number of lanes a value lives in -- 15 + 1 shuffles and adds (plus selects) instead of 16 x 5.  Returns, in EVERY lane, the
// warp-wide sum of v[(lane >> 1) & 15].  Fixed association order (deterministic).
__device__ __forceinline__ float warp_sum16_transposed(const float (&v)[16], int lane) {
    float a[8], b[4], c[2];
    bool up = (lane & 16) != 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = (up ? v[i + 8] : v[i]) + __shfl_xor_sync(0xffffffffu, up ? v[i] : v[i + 8], 16);
    up = (lane & 8) != 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) b[i] = (up ? a[i + 4] : a[i]) + __shfl_xor_sync(0xffffffffu, up ? a[i] : a[i + 4], 8);
    up = (lane & 4) != 0;
#pragma unroll
    for (int i = 0; i < 2; ++i) c[i] = (up ? b[i + 2] : b[i]) + __shfl_xor_sync(0xffffffffu, up ? b[i] : b[i + 2], 4);
    up = (lane & 2) != 0;
    float d = (up ? c[1] : c[0]) + __shfl_xor_sync(0xffffffffu, up ? c[0] : c[1], 2);
    d += __shfl_xor_sync(0xffffffffu, d, 1);
    return d;
}

struct ThreadId {
    int t, warp, lane, m, wx, wy;
    bool worker;
    __device__ __forceinline__ ThreadId() : ThreadId((int)threadIdx.x) {}
    // thread tt of a 224-thread group (one image's threads)
    __device__ __forceinline__ explicit ThreadId(int tt) {
        t = tt;
        warp = t >> 5;
        lane = t & 31;
        worker = t < NWK;
        m = worker ? t / 36 : 0;
        wx = worker ? (t % 36) / 6 : 0;
        wy = worker ? t % 6 : 0;
    }
};

// register-resident accumulators of one thread, kept across all images a CTA processes in one step
struct Acc {
    float dw_c1[25], dw_s1[16], dw_f[PCNN_F];
    float bsum_c1, bsum_s1, gfb, err_acc;
    int wrong;
    __device__ __forceinline__ void zero() {
#pragma unroll
        for (int i = 0; i < 25; ++i) dw_c1[i] = 0.0f;
#pragma unroll
        for (int i = 0; i < 16; ++i) dw_s1[i] = 0.0f;
#pragma unroll
        for (int i = 0; i < PCNN_F; ++i) dw_f[i] = 0.0f;
        bsum_c1 = bsum_s1 = gfb = err_acc = 0.0f;
        wrong = 0;
    }
};

// H1: the second image's buffers of a two-image CTA, else null
template <typename InT> __device__ __forceinline__ void init_barriers(FusedSmem<InT> &S, ImageSmem<InT> *H1 = nullptr) {
    if (threadIdx.x == 0) {
        mbar_init(&S.mbar[0], 1);
        mbar_init(&S.mbar[1], 1);
        mbar_init(&S.params_bar, 1);
        mbar_init(&S.grads_bar, 1);
        if (H1) {
            mbar_init(&H1->mbar[0], 1);
            mbar_init(&H1->mbar[1], 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // mnist.h:145 + Main.cpp:64: (float)((double)u / 255.0).  u / 255 has a period-8 binary expansion, so rounding the exact
    // quotient straight to fp32 equals rounding via double (checked for all 256 values in tests/); one table per CTA instead
    // of four IEEE divisions per thread and image
    for (int u = threadIdx.x; u < 256; u += blockDim.x) S.lut[u] = __fdiv_rn((float)u, 255.0f);
    __syncthreads();
}

// thread 0 of the image's threads only: start the bulk copy of one image into staging buffer `buf`
template <typename InT> __device__ __forceinline__ void issue_image(ImageSmem<InT> &H, int buf, const InT *src) {
    constexpr bool IS_U8 = (sizeof(InT) == 1);
    constexpr unsigned IMG_BYTES = PCNN_IMG * sizeof(InT);
    mbar_expect_tx(&H.mbar[buf], IMG_BYTES);
    bulk_g2s(IS_U8 ? (void *)H.stage[buf] : (void *)H.imgf[buf], src, IMG_BYTES, &H.mbar[buf]);
}
// thread 0 only: start the bulk copy of the packed parameters
template <typename InT> __device__ __forceinline__ void issue_params(FusedSmem<InT> &S, const float *params) {
    mbar_expect_tx(&S.params_bar, NPACK * 4);
    bulk_g2s(S.params, params, NPACK * 4, &S.params_bar);
}

// hook called by thread 0 right before it issues the bulk copy of a prefetched image (the persistent kernel gates on the
// arrival of host-streamed chunks there); the default does nothing
struct NoGate {
    __device__ __forceinline__ void operator()(const void *) const {}
};

struct EvalOut {
    float *f_out;     // this image's 10 outputs or null
    uint8_t *pred;    // this image's prediction or null
    bool has_label;
};

// One image through the CTA.  `li` is the CTA-local running image counter (selects the staging buffer and the mbarrier
// phase); the image must have been issued into buffer li & 1.  `next_src` (or null) is prefetched into the other buffer
// right after the first barrier.  `params_parity` < 0: parameters already resident; otherwise wait on mbar[2] with that
// parity before the first use of S.params (lets the parameter copy overlap the u8 -> fp32 conversion).
// P0 of an image: wait until it has landed in staging buffer li & 1, convert it to fp32 (u8 path), fetch the label.  No
// barrier: the caller's next block barrier (sync #1 of image_pass) publishes the results.
// H: the image's buffers (S itself, or the second image's of a two-image CTA).
template <typename InT>
__device__ __forceinline__ void image_prepare(FusedSmem<InT> &S, ImageSmem<InT> &H, const ThreadId &id, int li, const uint8_t *label_ptr) {
    constexpr bool IS_U8 = (sizeof(InT) == 1);
    const int t = id.t;
    const int buf = li & 1;
    mbar_wait(&H.mbar[buf], (unsigned)(li >> 1) & 1u);
    if (IS_U8) {
        if (t < 196) {
            uchar4 q = reinterpret_cast<const uchar4 *>(H.stage[buf])[t];
            float4 f = make_float4(S.lut[q.x], S.lut[q.y], S.lut[q.z], S.lut[q.w]);
            reinterpret_cast<float4 *>(H.imgf[buf])[t] = f;
        }
    }
    if (t == NWK && label_ptr) H.label[buf] = (int)*label_ptr;
}

// `prepared`: image_prepare has already run for this image (the persistent kernel does it while it waits for the step's
// parameters).
template <typename InT, bool TRAIN, typename Gate = NoGate>
__device__ __forceinline__ void image_pass(FusedSmem<InT> &S, const ThreadId &id, int li, const uint8_t *label_ptr,
                                           const InT *next_src, int params_parity, Acc &A, const EvalOut &ev,
                                           const Gate &gate = Gate(), bool prepared = false) {
    const int t = id.t, warp = id.warp, lane = id.lane;
    const int buf = li & 1;
    // ---- P0: the image has landed; convert to fp32 (u8 path), fetch the label
    if (!prepared) image_prepare(S, S, id, li, label_ptr);
    if (params_parity >= 0) mbar_wait(&S.params_bar, (unsigned)params_parity);
    __syncthreads();                                                         // sync #1
    if (t == 0 && next_src) {
        gate(next_src);
        issue_image(S, buf ^ 1, next_src);
    }
    // Single-lane blocks (TMA issue by lane 0 of warp 0, label fetch by lane 24 of warp 6) leave their warp diverged:
    // ptxas places the reconvergence point far downstream, and the butterfly shuffles below were then executed by
    // a partial warp (observed once: warp 0's FC partial sums lost lane 0).  Reconverge explicitly.
    __syncwarp();

    // ---- P1: c1 (5x5 valid conv, layer.h:105-140) + sigmoid, s1 (4x4/4 weighted sum, layer.h:143-181) + sigmoid
    float o[16];         // this worker's 4x4 block of c1 outputs
    float s1o = 0.0f;    // its s1 output
    float fcp[PCNN_F];
    float fw[PCNN_F];    // this worker's column of f.weight, used again by the backward chain
#pragma unroll
    for (int q = 0; q < PCNN_F; ++q) fcp[q] = fw[q] = 0.0f;
    if (id.worker) {
        // Filter row i outermost: its five weights and one 8-wide patch row are all that is live next to the 16
        // accumulators (the whole 8x8 patch or all 25 weights in registers do not fit beside the gradient accumulators).
        // Every accumulator still receives its 25 terms in (i, j) order.
        const float *ip = S.imgf[buf] + (4 * id.wx) * 28 + 4 * id.wy;
        float acc[16];
#pragma unroll
        for (int p = 0; p < 16; ++p) acc[p] = 0.0f;
        const float *wc = S.params + OFF_C1W + id.m * 25;
#pragma unroll
        for (int i = 0; i < 5; ++i) {
            float w[5];
#pragma unroll
            for (int j = 0; j < 5; ++j) w[j] = wc[i * 5 + j];
#pragma unroll
            for (int ox = 0; ox < 4; ++ox) {
                const float4 lo = *reinterpret_cast<const float4 *>(ip + (ox + i) * 28);
                const float4 hi = *reinterpret_cast<const float4 *>(ip + (ox + i) * 28 + 4);
                const float x[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
                for (int j = 0; j < 5; ++j)
#pragma unroll
                    for (int oy = 0; oy < 4; ++oy) acc[ox * 4 + oy] = fmaf(x[oy + j], w[j], acc[ox * 4 + oy]);
            }
        }
        const float bc = S.params[OFF_C1B + id.m];
        float s1pre = 0.0f;
#pragma unroll
        for (int p = 0; p < 16; ++p) {
            o[p] = sigmoid_fast(acc[p] + bc);
            s1pre = fmaf(S.params[OFF_S1W + p], o[p], s1pre);
        }
        s1o = sigmoid_fast(s1pre + S.params[OFF_S1B]);
        // fp_preact_f partial products (layer.h:184-203): this worker owns input k = t
#pragma unroll
        for (int q = 0; q < PCNN_F; ++q) {
            fw[q] = S.params[OFF_FW + q * PCNN_S1 + t];
            fcp[q] = fw[q] * s1o;
        }
    } else {
#pragma unroll
        for (int p = 0; p < 16; ++p) o[p] = 0.0f;
    }
    __syncwarp();                                                            // workers / helpers of warp 6 rejoin
#pragma unroll
    for (int q = 0; q < PCNN_F; ++q) {
        float v = warp_sum(fcp[q]);
        if (lane == 0) S.fc_red[warp][q] = v;
    }
    __syncthreads();                                                         // sync #2

    // ---- P2: f layer output, makeError (layer.h:91-95), vectorNorm (Main.cpp:28-34)
    float dq[PCNN_F];    // TRAIN: d_preact of the f layer, in every thread
    if (TRAIN) {
        // Every warp finishes the ten outputs itself (lanes 0..9; 7 + 1 adds, one sigmoid) and broadcasts d_preact by
        // shuffle: no third block barrier and no shared-memory round trip; warp 0 also keeps the bias / error sums.
        float d = 0.0f;
        if (lane < PCNN_F) {
            float pre = 0.0f;
#pragma unroll
            for (int w = 0; w < NWARP; ++w) pre += S.fc_red[w][lane];
            pre += S.params[OFF_FB + lane];                                  // fp_bias_f, layer.h:206-211
            const float outv = sigmoid_fast(pre);
            d = (lane == S.label[buf] ? 1.0f : 0.0f) - outv;
        }
        __syncwarp();
#pragma unroll
        for (int q = 0; q < PCNN_F; ++q) dq[q] = __shfl_sync(0xffffffffu, d, q);
        if (warp == 0) {
            A.gfb += d;                                                      // lanes >= 10 add zero
            float ss = 0.0f;
#pragma unroll
            for (int q = 0; q < PCNN_F; ++q) ss = fmaf(dq[q], dq[q], ss);
            A.err_acc += sqrtf(ss);                                          // every lane holds the same value; lane 0's is used
        }
    } else {
        if (warp == 0) {
            float outv = 0.0f;
            if (lane < PCNN_F) {
                float pre = 0.0f;
#pragma unroll
                for (int w = 0; w < NWARP; ++w) pre += S.fc_red[w][lane];
                pre += S.params[OFF_FB + lane];
                outv = sigmoid_fast(pre);
                S.f_out[lane] = outv;
                if (ev.f_out) ev.f_out[lane] = outv;
            }
            __syncwarp();
            if (lane == 0) {                                                 // classify(), Main.cpp:193-197
                int best = 0;
#pragma unroll
                for (int q = 1; q < PCNN_F; ++q)
                    if (S.f_out[best] < S.f_out[q]) best = q;
                if (ev.pred) *ev.pred = (uint8_t)best;
                if (ev.has_label && best != S.label[buf]) ++A.wrong;
            }
        }
        return;   // the next image's sync #1 orders the reuse of fc_red / f_out
    }

    // ---- P3: backward chain (Main.cpp:114-131)
    if (id.worker) {
        float dout_s1 = 0.0f;
#pragma unroll
        for (int q = 0; q < PCNN_F; ++q) {
            A.dw_f[q] = fmaf(dq[q], s1o, A.dw_f[q]);                                       // bp_weight_f, layer.h:214-227
            dout_s1 = fmaf(fw[q], dq[q], dout_s1);                                          // bp_output_s1, layer.h:237-257
        }
        const float dpre_s1 = dout_s1 * s1o * (1.0f - s1o);                                // bp_preact_s1, layer.h:260-270
        A.bsum_s1 += dpre_s1;                                                               // bp_bias_s1 accumulator, layer.h:303-314
        float dpc[16];
        float bs = 0.0f;
#pragma unroll
        for (int p = 0; p < 16; ++p) {
            A.dw_s1[p] = fmaf(dpre_s1, o[p], A.dw_s1[p]);                                   // bp_weight_s1, layer.h:272-300
            const float dout_c1 = S.params[OFF_S1W + p] * dpre_s1;                          // bp_output_c1, layer.h:319-346
            dpc[p] = dout_c1 * (o[p] * (1.0f - o[p]));                                      // bp_preact_c1, layer.h:348-369
            bs += dpc[p];
        }
        A.bsum_c1 += bs;                                                                    // bp_bias_c1 accumulator, layer.h:400-410
        // bp_weight_c1, layer.h:371-395 (the /576 is applied once in the epilogue)
        const float *ip = S.imgf[buf] + (4 * id.wx) * 28 + 4 * id.wy;
#pragma unroll
        for (int i = 0; i < 5; ++i) {
#pragma unroll
            for (int ox = 0; ox < 4; ++ox) {
                const float4 lo = *reinterpret_cast<const float4 *>(ip + (ox + i) * 28);
                const float4 hi = *reinterpret_cast<const float4 *>(ip + (ox + i) * 28 + 4);
                const float x[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
                for (int j = 0; j < 5; ++j)
#pragma unroll
                    for (int oy = 0; oy < 4; ++oy) A.dw_c1[i * 5 + j] = fmaf(dpc[ox * 4 + oy], x[oy + j], A.dw_c1[i * 5 + j]);
            }
        }
    }
}

// Reduce the register accumulators of the 216 workers in a fixed order and write this CTA's packed partial gradient
// (slot[NPACK]).  Ends with all of the CTA's global stores issued (callers fence as needed).
// plain fp32 slot (graph path) / tagged words (persistent kernel)
struct FloatSink {
    float *slot;
    __device__ __forceinline__ void operator()(int p, float v) const { slot[p] = v; }
};
struct SmemSink {
    float *dst;
    __device__ __forceinline__ void operator()(int p, float v) const { dst[p] = v; }
};
struct LLSink {
    llword *slot;
    unsigned tag;
    __device__ __forceinline__ void operator()(int p, float v) const { ll_store(slot + p, v, tag); }
};

template <typename InT, typename Sink>
__device__ __forceinline__ void cta_epilogue(FusedSmem<InT> &S, const ThreadId &id, const Acc &A, const Sink &put) {
    const int t = id.t, warp = id.warp, lane = id.lane;
    __syncthreads();
    if (id.worker) {
#pragma unroll
        for (int i = 0; i < 25; ++i) S.red[t * RED_STRIDE + i] = A.dw_c1[i];
        S.red[t * RED_STRIDE + 25] = A.bsum_c1;
#pragma unroll
        for (int q = 0; q < PCNN_F; ++q) put(OFF_FW + q * PCNN_S1 + t, A.dw_f[q]);   // column t is private to this worker
    }
    __syncwarp();
#pragma unroll
    for (int p = 0; p < 16; ++p) {
        float v = warp_sum(A.dw_s1[p]);
        if (lane == 0) S.red_s1[warp][p] = v;
    }
    {
        float v = warp_sum(A.bsum_s1);
        if (lane == 0) S.red_s1[warp][16] = v;
    }
    __syncthreads();
    if (t < 156) {                       // 150 c1 taps + 6 c1 bias sums: sum over the 36 windows of a map, 4 chains
        const int mm = t < 150 ? t / 25 : t - 150;
        const int col = t < 150 ? t % 25 : 25;
        const float *r = S.red + (mm * 36) * RED_STRIDE + col;
        float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
#pragma unroll
        for (int w = 0; w < 36; w += 4) {
            s0 += r[(w + 0) * RED_STRIDE];
            s1 += r[(w + 1) * RED_STRIDE];
            s2 += r[(w + 2) * RED_STRIDE];
            s3 += r[(w + 3) * RED_STRIDE];
        }
        const float s = (s0 + s1) + (s2 + s3);
        if (t < 150) put(OFF_C1W + t, s * (1.0f / 576.0f));
        else put(OFF_C1B + mm, s);
    } else if (t < 173) {                // s1 taps and s1 bias sum
        const int p = t - 156;
        float s = 0.0f;
#pragma unroll
        for (int w = 0; w < NWARP; ++w) s += S.red_s1[w][p];
        put(OFF_S1W + p, s);             // p == 16 lands on OFF_S1B
    }
    if (t < PCNN_F) put(OFF_FB + t, A.gfb);
    if (t == 0) put(OFF_ERR, A.err_acc);
}

// ----------------------------------------------------------------------------------------------------------------------
// One image per CTA and step (batch <= grid: the configuration BASELINE.json quotes its metric on): forward + backward + CTA
// reduction in one piece, specialised on the fact that nothing is accumulated across images:
//   * the gradient accumulators are not live during the forward pass, so the worker's WHOLE 8x8 input patch stays in
//     registers from the forward convolution to the weight gradient -- no shared-memory operand inside either FFMA block;
//   * the f-layer weight gradient (2,160 of the 2,344 packed entries) is pushed to its consumers right after the f layer,
//     BEFORE the backward convolution, and the s1 sums are reduced there too: what remains for the end of the pass are the
//     156 c1 entries.
// `put(p, v)` consumes packed entry p (the persistent kernel pushes it to the cluster rank that owns it).  The image must
// have been prepared (image_prepare) by the caller; `S.params` must be complete.  Same arithmetic as image_pass + cta_epilogue.
//
// IPC = 2: a 448-thread CTA trains two images side by side, threads half * 224 + id.t running image `half` out of its own
// buffers H with the arithmetic above; both halves read the one S.params.  Half 1 hands its f-layer gradient, f bias / error
// and end-of-pass sums to half 0 through X (named barriers 1 and 2, arrive / sync: half 1 never waits), and half 0 pushes
// image 0 + image 1 of every packed entry, once per CTA.
template <int IPC, typename InT, typename Sink>
__device__ __forceinline__ void image_step_single(FusedSmem<InT> &S, ImageSmem<InT> &H, PairXchg *X, const ThreadId &id, int half, int li,
                                                  bool has_image, const Sink &put) {
    constexpr bool PAIR = IPC == 2;
    const int t = id.t, warp = id.warp, lane = id.lane;
    const int buf = li & 1;
    __syncthreads();                                                         // sync #1: image + parameters visible
    const bool work = id.worker && has_image;
    float o[16];
    float s1o = 0.0f;
    float fcp[16], fw[PCNN_F];          // fcp: ten partial products, padded to the sixteen of the transposed warp sum
#pragma unroll
    for (int q = 0; q < 16; ++q) fcp[q] = 0.0f;
#pragma unroll
    for (int q = 0; q < PCNN_F; ++q) fw[q] = 0.0f;
#pragma unroll
    for (int p = 0; p < 16; ++p) o[p] = 0.0f;
    const float *ip = H.imgf[buf] + (id.worker ? (4 * id.wx) * 28 + 4 * id.wy : 0);
    if (work) {
        float patch[8][8];
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            const float4 lo = *reinterpret_cast<const float4 *>(ip + r * 28);
            const float4 hi = *reinterpret_cast<const float4 *>(ip + r * 28 + 4);
            patch[r][0] = lo.x; patch[r][1] = lo.y; patch[r][2] = lo.z; patch[r][3] = lo.w;
            patch[r][4] = hi.x; patch[r][5] = hi.y; patch[r][6] = hi.z; patch[r][7] = hi.w;
        }
        float acc[16];
#pragma unroll
        for (int p = 0; p < 16; ++p) acc[p] = 0.0f;
        const float *wc = S.params + OFF_C1W + id.m * 25;
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
            for (int j = 0; j < 5; ++j) {                                    // fp_c1, layer.h:105-140: terms in (i, j) order
                const float w = wc[i * 5 + j];
#pragma unroll
                for (int ox = 0; ox < 4; ++ox)
#pragma unroll
                    for (int oy = 0; oy < 4; ++oy) acc[ox * 4 + oy] = fmaf(patch[ox + i][oy + j], w, acc[ox * 4 + oy]);
            }
        const float bc = S.params[OFF_C1B + id.m];
        float s1pre = 0.0f;
#pragma unroll
        for (int p = 0; p < 16; ++p) {
            o[p] = sigmoid_fast(acc[p] + bc);
            s1pre = fmaf(S.params[OFF_S1W + p], o[p], s1pre);                // fp_s1, layer.h:143-181
        }
        s1o = sigmoid_fast(s1pre + S.params[OFF_S1B]);
#pragma unroll
        for (int q = 0; q < PCNN_F; ++q) {                                   // fp_preact_f partial products, layer.h:184-203
            fw[q] = S.params[OFF_FW + q * PCNN_S1 + t];
            fcp[q] = fw[q] * s1o;
        }
    }
    __syncwarp();
    {
        const float v = warp_sum16_transposed(fcp, lane);                    // lane 2q (and 2q + 1) holds output q's warp sum
        if ((lane & 1) == 0 && (lane >> 1) < PCNN_F) H.fc_red[warp][lane >> 1] = v;
    }
    __syncthreads();                                                         // sync #2
    // f output, makeError (layer.h:91-95), vectorNorm (Main.cpp:28-34): every warp for itself, d_preact broadcast by shuffle
    float dq[PCNN_F];
    float d = 0.0f;
    if (lane < PCNN_F && has_image) {
        float pre = 0.0f;
#pragma unroll
        for (int w = 0; w < NWARP; ++w) pre += H.fc_red[w][lane];
        pre += S.params[OFF_FB + lane];                                      // fp_bias_f, layer.h:206-211
        d = (lane == H.label[buf] ? 1.0f : 0.0f) - sigmoid_fast(pre);
    }
    __syncwarp();
#pragma unroll
    for (int q = 0; q < PCNN_F; ++q) dq[q] = __shfl_sync(0xffffffffu, d, q);
    float err = 0.0f;
    if (!PAIR) {
        if (warp == 0) {
            if (lane < PCNN_F) put(OFF_FB + lane, d);                        // bp_bias_f accumulator, layer.h:229-234
            if (lane == 0) {
                float ss = 0.0f;
#pragma unroll
                for (int q = 0; q < PCNN_F; ++q) ss = fmaf(dq[q], dq[q], ss);
                put(OFF_ERR, has_image ? sqrtf(ss) : 0.0f);
            }
        }
    } else if (warp == 0 && lane == 0) {
        float ss = 0.0f;
#pragma unroll
        for (int q = 0; q < PCNN_F; ++q) ss = fmaf(dq[q], dq[q], ss);
        err = has_image ? sqrtf(ss) : 0.0f;
    }
    if (PAIR && half == 1) {                                                  // image 1's f-layer entries go to half 0
        if (warp == 0) {
            if (lane < PCNN_F) X->fb[lane] = d;
            if (lane == 0) X->fb[PCNN_F] = err;
        }
        if (id.worker) {
#pragma unroll
            for (int q = 0; q < PCNN_F; ++q) X->fw[q][t] = dq[q] * s1o;
        }
        __syncwarp();
        named_bar_arrive(1, 2 * NT);
    } else if (PAIR) {                                                       // image 0 + image 1, before the convolution
        __syncwarp();
        named_bar_sync(1, 2 * NT);
        if (warp == 0) {
            if (lane < PCNN_F) put(OFF_FB + lane, d + X->fb[lane]);
            if (lane == 0) put(OFF_ERR, err + X->fb[PCNN_F]);
        }
    }
    __syncwarp();
    // backward chain (Main.cpp:114-131)
    float dpc[16], dws[17];
    float bsum_c1 = 0.0f;
#pragma unroll
    for (int p = 0; p < 16; ++p) dpc[p] = 0.0f;
#pragma unroll
    for (int p = 0; p < 17; ++p) dws[p] = 0.0f;
    if (id.worker) {
        float dout_s1 = 0.0f;
#pragma unroll
        for (int q = 0; q < PCNN_F; ++q) {
            if (!PAIR) put(OFF_FW + q * PCNN_S1 + t, dq[q] * s1o);           // bp_weight_f, layer.h:214-227: on its way already
            else if (half == 0) put(OFF_FW + q * PCNN_S1 + t, __fmul_rn(dq[q], s1o) + X->fw[q][t]);
            dout_s1 = fmaf(fw[q], dq[q], dout_s1);                           // bp_output_s1, layer.h:237-257
        }
        const float dpre_s1 = dout_s1 * s1o * (1.0f - s1o);                  // bp_preact_s1, layer.h:260-270
        dws[16] = dpre_s1;                                                   // bp_bias_s1 accumulator, layer.h:303-314
#pragma unroll
        for (int p = 0; p < 16; ++p) {
            dws[p] = dpre_s1 * o[p];                                         // bp_weight_s1, layer.h:272-300
            const float dout_c1 = S.params[OFF_S1W + p] * dpre_s1;           // bp_output_c1, layer.h:319-346
            dpc[p] = dout_c1 * (o[p] * (1.0f - o[p]));                       // bp_preact_c1, layer.h:348-369
            bsum_c1 += dpc[p];                                               // bp_bias_c1 accumulator, layer.h:400-410
        }
    }
    __syncwarp();
    {                                                                        // s1 sums: warp level now, across warps at the end
        float d16[16];
#pragma unroll
        for (int p = 0; p < 16; ++p) d16[p] = dws[p];
        const float v = warp_sum16_transposed(d16, lane);
        if ((lane & 1) == 0) H.red_s1[warp][lane >> 1] = v;
        const float vb = warp_sum(dws[16]);
        if (lane == 0) H.red_s1[warp][16] = vb;
    }
    if (id.worker) {
        // bp_weight_c1, layer.h:371-395 (the /576 is applied once, below): the patch comes back from shared memory in one go
        // (16 loads), so the FFMA block below has register operands only
        float patch[8][8];
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            const float4 lo = *reinterpret_cast<const float4 *>(ip + r * 28);
            const float4 hi = *reinterpret_cast<const float4 *>(ip + r * 28 + 4);
            patch[r][0] = lo.x; patch[r][1] = lo.y; patch[r][2] = lo.z; patch[r][3] = lo.w;
            patch[r][4] = hi.x; patch[r][5] = hi.y; patch[r][6] = hi.z; patch[r][7] = hi.w;
        }
        float *row = H.red + t * RED_STRIDE;
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
        row[25] = bsum_c1;
    }
    __syncthreads();                                                         // sync #3: H.red, H.red_s1 complete
    if (!PAIR) {
        if (t < 156) {                   // 150 c1 taps + 6 c1 bias sums: sum over the 36 windows of a map, 4 chains
            const int mm = t < 150 ? t / 25 : t - 150;
            const int col = t < 150 ? t % 25 : 25;
            const float *r = H.red + (mm * 36) * RED_STRIDE + col;
            float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
#pragma unroll
            for (int w = 0; w < 36; w += 4) {
                s0 += r[(w + 0) * RED_STRIDE];
                s1 += r[(w + 1) * RED_STRIDE];
                s2 += r[(w + 2) * RED_STRIDE];
                s3 += r[(w + 3) * RED_STRIDE];
            }
            const float ssum = (s0 + s1) + (s2 + s3);
            if (t < 150) put(OFF_C1W + t, ssum * (1.0f / 576.0f));
            else put(OFF_C1B + mm, ssum);
        } else if (t < 173) {            // s1 taps and s1 bias sum
            const int p = t - 156;
            float ssum = 0.0f;
#pragma unroll
            for (int w = 0; w < NWARP; ++w) ssum += H.red_s1[w][p];
            put(OFF_S1W + p, ssum);      // p == 16 lands on OFF_S1B
        }
        return;
    }
    // the same sums of both images: image 0 + image 1
    float ssum = 0.0f;
    if (t < 156) {
        const int mm = t < 150 ? t / 25 : t - 150;
        const int col = t < 150 ? t % 25 : 25;
        const float *r = H.red + (mm * 36) * RED_STRIDE + col;
        float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
#pragma unroll
        for (int w = 0; w < 36; w += 4) {
            s0 += r[(w + 0) * RED_STRIDE];
            s1 += r[(w + 1) * RED_STRIDE];
            s2 += r[(w + 2) * RED_STRIDE];
            s3 += r[(w + 3) * RED_STRIDE];
        }
        ssum = (s0 + s1) + (s2 + s3);
    } else if (t < 173) {
#pragma unroll
        for (int w = 0; w < NWARP; ++w) ssum += H.red_s1[w][t - 156];
    }
    if (half == 1) {
        if (t < 173) X->tail[t] = ssum;
        __syncwarp();
        named_bar_arrive(2, 2 * NT);
        return;
    }
    __syncwarp();
    named_bar_sync(2, 2 * NT);                                               // the 72 windows / 14 warps of the pair
    if (t < 173) ssum += X->tail[t];
    if (t < 150) put(OFF_C1W + t, ssum * (1.0f / 576.0f));
    else if (t < 156) put(OFF_C1B + t - 150, ssum);
    else if (t < 173) put(OFF_S1W + t - 156, ssum);                          // t == 172 lands on OFF_S1B
}

// Several images per CTA and step (batch > grid): the same structure as image_step_single -- whole patch in registers per
// convolution, transposed warp sums -- with the batch sums kept where they cost least: the 25 + 1 c1 sums in registers, the
// f-layer weight gradient in thread-private shared memory (S.accf), the s1 sums in lane-private shared memory (S.red_s1),
// the f bias / error sums in warp 0's registers.  Images b = c, c + G, ... < nb; the first one has been prepared by the
// caller, the others are prefetched one ahead.  Returns the advanced image counter.
template <typename InT, typename Gate, typename Sink>
__device__ __forceinline__ int image_steps_multi(FusedSmem<InT> &S, const ThreadId &id, const InT *img_base, const uint8_t *lab_base, int c,
                                                 int G, int nb, int li, const Gate &gate, const Sink &put) {
    const int t = id.t, warp = id.warp, lane = id.lane;
    float dw_c1[25];
#pragma unroll
    for (int k = 0; k < 25; ++k) dw_c1[k] = 0.0f;
    float bsum_c1 = 0.0f, gfb = 0.0f, err_acc = 0.0f;
#pragma unroll
    for (int q = 0; q < PCNN_F; ++q) S.accf[q * NT + t] = 0.0f;              // thread-private
    if ((lane & 1) == 0) S.red_s1[warp][lane >> 1] = 0.0f;                   // lane-private
    if (lane == 0) S.red_s1[warp][16] = 0.0f;
    const float *ip_off = nullptr;
    for (int b = c; b < nb; b += G, ++li) {
        const int buf = li & 1;
        if (b != c) image_prepare(S, S, id, li, lab_base + b);
        __syncthreads();                                                     // sync #1: image (+ parameters) visible
        const int bn = b + G;
        if (t == 0 && bn < nb) {
            const InT *nsrc = img_base + (long long)bn * PCNN_IMG;
            gate(nsrc);
            issue_image(S, buf ^ 1, nsrc);
        }
        __syncwarp();
        float o[16];
        float s1o = 0.0f;
        float fcp[16], fw[PCNN_F];
#pragma unroll
        for (int q = 0; q < 16; ++q) fcp[q] = 0.0f;
#pragma unroll
        for (int q = 0; q < PCNN_F; ++q) fw[q] = 0.0f;
#pragma unroll
        for (int p = 0; p < 16; ++p) o[p] = 0.0f;
        const float *ip = S.imgf[buf] + (id.worker ? (4 * id.wx) * 28 + 4 * id.wy : 0);
        ip_off = ip;
        if (id.worker) {
            float patch[8][8];
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const float4 lo = *reinterpret_cast<const float4 *>(ip + r * 28);
                const float4 hi = *reinterpret_cast<const float4 *>(ip + r * 28 + 4);
                patch[r][0] = lo.x; patch[r][1] = lo.y; patch[r][2] = lo.z; patch[r][3] = lo.w;
                patch[r][4] = hi.x; patch[r][5] = hi.y; patch[r][6] = hi.z; patch[r][7] = hi.w;
            }
            float acc[16];
#pragma unroll
            for (int p = 0; p < 16; ++p) acc[p] = 0.0f;
            const float *wc = S.params + OFF_C1W + id.m * 25;
#pragma unroll
            for (int i = 0; i < 5; ++i)
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                    const float w = wc[i * 5 + j];
#pragma unroll
                    for (int ox = 0; ox < 4; ++ox)
#pragma unroll
                        for (int oy = 0; oy < 4; ++oy) acc[ox * 4 + oy] = fmaf(patch[ox + i][oy + j], w, acc[ox * 4 + oy]);
                }
            const float bc = S.params[OFF_C1B + id.m];
            float s1pre = 0.0f;
#pragma unroll
            for (int p = 0; p < 16; ++p) {
                o[p] = sigmoid_fast(acc[p] + bc);
                s1pre = fmaf(S.params[OFF_S1W + p], o[p], s1pre);
            }
            s1o = sigmoid_fast(s1pre + S.params[OFF_S1B]);
#pragma unroll
            for (int q = 0; q < PCNN_F; ++q) {
                fw[q] = S.params[OFF_FW + q * PCNN_S1 + t];
                fcp[q] = fw[q] * s1o;
            }
        }
        __syncwarp();
        {
            const float v = warp_sum16_transposed(fcp, lane);
            if ((lane & 1) == 0 && (lane >> 1) < PCNN_F) S.fc_red[warp][lane >> 1] = v;
        }
        __syncthreads();                                                     // sync #2
        float dq[PCNN_F];
        float d = 0.0f;
        if (lane < PCNN_F) {
            float pre = 0.0f;
#pragma unroll
            for (int w = 0; w < NWARP; ++w) pre += S.fc_red[w][lane];
            pre += S.params[OFF_FB + lane];
            d = (lane == S.label[buf] ? 1.0f : 0.0f) - sigmoid_fast(pre);
        }
        __syncwarp();
#pragma unroll
        for (int q = 0; q < PCNN_F; ++q) dq[q] = __shfl_sync(0xffffffffu, d, q);
        if (warp == 0) {
            gfb += d;
            float ss = 0.0f;
#pragma unroll
            for (int q = 0; q < PCNN_F; ++q) ss = fmaf(dq[q], dq[q], ss);
            err_acc += sqrtf(ss);
        }
        float dpc[16], dws[16];
        float dpre_s1 = 0.0f;
#pragma unroll
        for (int p = 0; p < 16; ++p) dpc[p] = dws[p] = 0.0f;
        if (id.worker) {
            float dout_s1 = 0.0f;
#pragma unroll
            for (int q = 0; q < PCNN_F; ++q) {
                S.accf[q * NT + t] = fmaf(dq[q], s1o, S.accf[q * NT + t]);   // bp_weight_f, layer.h:214-227
                dout_s1 = fmaf(fw[q], dq[q], dout_s1);
            }
            dpre_s1 = dout_s1 * s1o * (1.0f - s1o);
#pragma unroll
            for (int p = 0; p < 16; ++p) {
                dws[p] = dpre_s1 * o[p];
                const float dout_c1 = S.params[OFF_S1W + p] * dpre_s1;
                dpc[p] = dout_c1 * (o[p] * (1.0f - o[p]));
                bsum_c1 += dpc[p];
            }
        }
        __syncwarp();
        {
            const float v = warp_sum16_transposed(dws, lane);
            if ((lane & 1) == 0) S.red_s1[warp][lane >> 1] += v;
            const float vb = warp_sum(dpre_s1);
            if (lane == 0) S.red_s1[warp][16] += vb;
        }
        if (id.worker) {
            float patch[8][8];
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const float4 lo = *reinterpret_cast<const float4 *>(ip + r * 28);
                const float4 hi = *reinterpret_cast<const float4 *>(ip + r * 28 + 4);
                patch[r][0] = lo.x; patch[r][1] = lo.y; patch[r][2] = lo.z; patch[r][3] = lo.w;
                patch[r][4] = hi.x; patch[r][5] = hi.y; patch[r][6] = hi.z; patch[r][7] = hi.w;
            }
#pragma unroll
            for (int i = 0; i < 5; ++i)
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                    float sacc = dw_c1[i * 5 + j];
#pragma unroll
                    for (int ox = 0; ox < 4; ++ox)
#pragma unroll
                        for (int oy = 0; oy < 4; ++oy) sacc = fmaf(dpc[ox * 4 + oy], patch[ox + i][oy + j], sacc);
                    dw_c1[i * 5 + j] = sacc;
                }
        }
    }
    (void)ip_off;
    // ---- CTA reduction of the batch sums
    if (id.worker) {
#pragma unroll
        for (int q = 0; q < PCNN_F; ++q) put(OFF_FW + q * PCNN_S1 + t, S.accf[q * NT + t]);
        float *row = S.red + t * RED_STRIDE;
#pragma unroll
        for (int k = 0; k < 25; ++k) row[k] = dw_c1[k];
        row[25] = bsum_c1;
    }
    if (t < PCNN_F) put(OFF_FB + t, gfb);
    if (t == 0) put(OFF_ERR, err_acc);
    __syncthreads();
    if (t < 156) {
        const int mm = t < 150 ? t / 25 : t - 150;
        const int col = t < 150 ? t % 25 : 25;
        const float *r = S.red + (mm * 36) * RED_STRIDE + col;
        float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
#pragma unroll
        for (int w = 0; w < 36; w += 4) {
            s0 += r[(w + 0) * RED_STRIDE];
            s1 += r[(w + 1) * RED_STRIDE];
            s2 += r[(w + 2) * RED_STRIDE];
            s3 += r[(w + 3) * RED_STRIDE];
        }
        const float ssum = (s0 + s1) + (s2 + s3);
        if (t < 150) put(OFF_C1W + t, ssum * (1.0f / 576.0f));
        else put(OFF_C1B + mm, ssum);
    } else if (t < 173) {
        const int p = t - 156;
        float ssum = 0.0f;
#pragma unroll
        for (int w = 0; w < NWARP; ++w) ssum += S.red_s1[w][p];
        put(OFF_S1W + p, ssum);
    }
    return li;
}

// entry p of the packed vector: w += step * g in the reference's operand order (layer.h:99, :316, :412)
__device__ __forceinline__ float updated_entry(float w, int p, float g, float step) {
    if (p >= OFF_C1B && p < OFF_S1W) return w + step * g / 576.0f;
    if (p == OFF_S1B) return w + step * g / 216.0f;
    return w + step * g;
}

// rank_local == 0: all ranks index one shared split (rank r starts at cursor + r * B), the global batch is clamped at
// the end of the split.  rank_local == 1: every rank walks its OWN equally sized shard (pcnn_learn_host), so the
// per-rank batch is clamped and multiplied by world.
__device__ __forceinline__ long long effective_global_batch(long long cursor, bool have_cursor, long long n_total, int B,
                                                            int world, int rank_local) {
    long long gb = (long long)B * world;
    if (have_cursor) {
        long long left = n_total - cursor;
        if (rank_local) {
            if (left < B) gb = left * world;
        } else if (left < gb) {
            gb = left;
        }
    }
    return gb < 1 ? 1 : gb;
}

}  // namespace pcnn_fused
