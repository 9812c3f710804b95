// parallel-cnn_b200/csrc/pcnn_internal.h -- shared declarations of the libpcnn.so translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <map>
#include <tuple>

#include "../../include/pcnn.h"

#define PCNN_VERSION_NUMBER 200   /* 0.2.0 */

// Packed vectors on the device carry one extra float: the batch sum of per-sample error norms.
constexpr int NPARAM = PCNN_NPARAM;
constexpr int NPACK = NPARAM + 1;           // 2344 floats = 9376 B, a multiple of 16 B (bulk-copy granule)
constexpr int OFF_C1W = PCNN_OFF_C1W, OFF_C1B = PCNN_OFF_C1B, OFF_S1W = PCNN_OFF_S1W, OFF_S1B = PCNN_OFF_S1B,
              OFF_FW = PCNN_OFF_FW, OFF_FB = PCNN_OFF_FB, OFF_ERR = PCNN_NPARAM;

// Fused-step launch geometry (see fused_kernels.cu)
constexpr int FUSED_THREADS = 224;          // 216 workers (one per (map, 4x4 window)) + 8 helpers
constexpr int FUSED_WORKERS = 216;
constexpr int FUSED_CTAS_PER_SM = 2;
constexpr int PCNN_TRACE_STEPS = 256;      // steps per launch the persistent kernel can timestamp
constexpr int STEP_ERR_CAP = 4096;        // most steps one replayed graph may hold
constexpr int MAX_SLOTS = 148 * 4;          // upper bound on the fused grid (per-CTA partial-gradient slots)

struct pcnn_split_binding {
    const void *images = nullptr;           // device
    const uint8_t *labels = nullptr;        // device
    int pixel_type = PCNN_U8;
    long n = 0;
    void *owned_images = nullptr;           // non-null when uploaded through pcnn_dataset_upload
    void *owned_labels = nullptr;
    bool rank_local = false;                // true: this rank's private shard (no rank offset into it)
    bool host_resident = false;             // images are the device alias of pinned HOST memory (pcnn_learn_host pulls them)
};

// where one step takes its samples from
struct pcnn_step_src {
    const void *images = nullptr;
    const uint8_t *labels = nullptr;
    int pixel_type = PCNN_U8;
    long n_total = 0;
    long first = 0;                         // explicit start when !use_cursor
    bool use_cursor = false;                // start = device-side cursor (+ rank * B unless rank_local)
    bool rank_local = false;
};

struct pcnn_graph_key {
    int B, nsteps, world, pixel_type, rank_local;
    const void *images;
    const void *labels;                     // both pointers are baked into the captured kernel arguments
    long n;
    bool operator<(const pcnn_graph_key &o) const {
        return std::tie(B, nsteps, world, pixel_type, rank_local, images, labels, n) <
               std::tie(o.B, o.nsteps, o.world, o.pixel_type, o.rank_local, o.images, o.labels, o.n);
    }
};

struct pcnn_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int sm_count = 0, cc_major = 0, cc_minor = 0;
    size_t hbm_bytes = 0;
    float lr = 1.0E-01f;                    // dt, layer.h:12

    float *d_params = nullptr;              // [NPACK]
    float *d_grads = nullptr;               // [NPACK] packed gradient (+ error sum) of the last step
    float *d_slots = nullptr;               // [MAX_SLOTS][NPACK] per-CTA partial gradients
    double *d_err_total = nullptr;          // running sum of error norms (double)
    long long *d_cursor = nullptr;          // next global sample index for cursor-driven steps
    int *d_wrong = nullptr;                 // misclassification counter of pcnn_test
    float *d_step_err = nullptr;            // [STEP_ERR_CAP] ring of per-step error sums, indexed by *d_step_idx
    int *d_step_idx = nullptr;              // device-side step counter (advanced by every cursor-driven step)
    float *h_step_err = nullptr;            // pinned, per-step error sums of the last pcnn_learn_host epoch
    long h_step_err_cap = 0, step_err_count = 0;

    pcnn_split_binding split[2];

    // host staging for the *_host entry points (pinned)
    void *h_stage[2] = {nullptr, nullptr};
    void *d_stage[2] = {nullptr, nullptr};
    uint8_t *h_stage_lab[2] = {nullptr, nullptr};
    uint8_t *d_stage_lab[2] = {nullptr, nullptr};
    size_t stage_bytes = 0;
    long stage_cap_samples = 0;
    float *h_scalar = nullptr;              // pinned scratch for blocking scalar read-backs
    // single-launch host streaming (pcnn_learn_host, persistent mode): the whole epoch is staged in HBM chunk by chunk
    // while the kernel already trains on the chunks that have landed
    void *d_hs_images = nullptr;
    uint8_t *d_hs_labels = nullptr;
    unsigned *d_hs_ready = nullptr;         // [hs_ready_cap] chunk flags
    unsigned *h_hs_tag = nullptr;           // pinned source word of the flag copies
    size_t hs_image_bytes = 0;
    long hs_label_cap = 0, hs_ready_cap = 0;
    unsigned hs_serial = 0;
    bool hs_copies_first = false;           // launches block the host thread (CUDA_LAUNCH_BLOCKING, kernel-replay profilers)
    bool launch_blocking_env = false;       // CUDA_LAUNCH_BLOCKING=1 at context creation (keeps hs_copies_first across pcnn_persist_tune)
    bool hs_no_pull = false;          // pcnn_persist_tune bit 4: pinned host images go through the staged stream too (A/B)
    double *h_hs_done = nullptr;            // pinned {double error sum, unsigned tag} written by the kernel after its last step
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_copy[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};

    std::map<pcnn_graph_key, cudaGraphExec_t> graphs;

    // data parallel state
    void *nccl_comm = nullptr;
    int rank = 0, world = 1;

    // persistent-kernel state (persist_kernels.cu)
    int step_mode = PCNN_MODE_AUTO;
    int persist_cap = 0;                    // co-resident CTAs of k_train_persist on this device
    bool persist_used = false;
    int persist_cluster_cap = 0;            // co-resident CTAs when launched as clusters of 8
    bool persist_no_coop = false;           // launch without the cooperative attribute (driver refusal or pcnn_persist_tune bit 1)
    bool persist_coop_refused = false;      // the driver refused a cooperative + cluster launch (keeps persist_no_coop across tunes)
    int persist_force_cluster = 0;          // > 0: cap the cluster size (A/B measurements through pcnn_persist_tune)
    int persist_last_cluster = 0, persist_last_grid = 0, persist_last_direct = 0;
    int persist_pair_cap[2] = {0, 0};       // co-resident two-image CTAs (448 threads) in clusters of 4 / of 2
    int persist_last_ipc = 0;               // images per CTA of the most recent launch
    bool persist_no_direct = false;         // measurement knob: keep the two-stage exchange on 2..4 GPUs
    int *d_abort = nullptr;                 // set by a spin loop that ran out of budget
    long long *d_trace = nullptr;           // optional phase timestamps of the persistent kernel (pcnn_persist_trace)
    unsigned p2p_step_id = 0;               // distributed steps issued since pcnn_p2p_attach (tags of the peer exchange)
    unsigned ll_step_id = 0;                // tags of the slot / parameter words (unique per context lifetime)
    unsigned long long *d_slots_ll = nullptr;   // [MAX_SLOTS][NPACK] tagged per-CTA partial gradients
    unsigned long long *d_params_ll = nullptr;  // [NPACK] tagged parameters
    void *p2p_base = nullptr;               // this rank's inbox + flags (IPC-exported)
    bool p2p_ready = false;
    uint2 *p2p_inbox = nullptr;             // [2][PCNN_MAX_PEERS][NPACK] words {value bits, step id}
    uint2 *p2p_peer_inbox[PCNN_MAX_PEERS] = {};
    void *p2p_mapped[PCNN_MAX_PEERS] = {};

    // grow-only device scratch of the convolution backward passes (partial sums, filter variants); stream-ordered reuse
    void *scratch = nullptr;
    size_t scratch_bytes = 0;
    void *scratch2 = nullptr;               // padded operands of the convolution backward passes (conv_bwd.cu)
    size_t scratch2_bytes = 0;

    int conv_bwd_path = PCNN_CONV_BWD_TENSOR;   // pcnn_conv_bwd_select

    long launches = 0;
};

// destroy every cached step graph (anything a captured kernel argument depends on has changed)
inline void pcnn_drop_graphs(pcnn_ctx *ctx) {
    for (auto &kv : ctx->graphs) cudaGraphExecDestroy(kv.second);
    ctx->graphs.clear();
}

// ---- error plumbing ------------------------------------------------------------------------------------
void pcnn_set_error(const char *fmt, ...);
int pcnn_fail_cuda(cudaError_t e, const char *what, const char *file, int line);

#define PCNN_CUDA(expr)                                                          \
    do {                                                                         \
        cudaError_t e__ = (expr);                                                \
        if (e__ != cudaSuccess) return pcnn_fail_cuda(e__, #expr, __FILE__, __LINE__); \
    } while (0)
#define PCNN_REQUIRE(cond, code, ...)                                            \
    do {                                                                         \
        if (!(cond)) { pcnn_set_error(__VA_ARGS__); return (code); }             \
    } while (0)
// the activation codes (PCNN_ACT_* of pcnn.h) every create call and pcnn_conv_bias_act_bwd take; any other is refused with
// this message, `fn` naming the called function
#define PCNN_REQUIRE_ACT(fn, act)                                                                                              \
    PCNN_REQUIRE((act) == PCNN_ACT_NONE || (act) == PCNN_ACT_SIGMOID || (act) == PCNN_ACT_RELU, PCNN_ERR_ARG,                 \
                 "%s: act %d is not 0 (none), 1 (sigmoid) or 3 (ReLU)", fn, act)
// column of a kernel table with one instantiation per activation: none, sigmoid, ReLU
inline int pcnn_act_col(int act) { return act == PCNN_ACT_RELU ? 2 : act; }
#define PCNN_CHECK_LAUNCH(ctx)                                                   \
    do {                                                                         \
        (ctx)->launches++;                                                       \
        cudaError_t e__ = cudaGetLastError();                                    \
        if (e__ != cudaSuccess) return pcnn_fail_cuda(e__, "kernel launch", __FILE__, __LINE__); \
    } while (0)

struct pcnn_device_guard {
    int prev = -1;
    explicit pcnn_device_guard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
    ~pcnn_device_guard() { if (prev >= 0) cudaSetDevice(prev); }
};

// ---- internal launchers shared between translation units -------------------------------------------------
// fused_kernels.cu
int pcnn_fused_configure();
int pcnn_launch_fused_grad(pcnn_ctx *ctx, const pcnn_step_src &src, int B, int *grid_out);
int pcnn_launch_reduce(pcnn_ctx *ctx, int grid_slots, int B, const pcnn_step_src &src, bool update, bool record_err);
int pcnn_launch_update(pcnn_ctx *ctx, int B, const pcnn_step_src &src, bool record_err);
// persist_kernels.cu
int pcnn_persist_configure(pcnn_ctx *ctx);
// Host streaming: the staged samples are cut into chunk 0 = [0, first) (one batch: the first step starts after a few
// microseconds of DMA), then kc chunks that double in size starting at c1 samples, then chunks of cmax samples -- short
// calls get few, soon-available chunks, long calls amortise the per-copy cost.  The samples of chunk k are readable once
// flags[k] == tag.  One function maps a sample to its chunk on both sides.
struct pcnn_chunking {
    long long first, c1, cmax;
    int kc;
};
__host__ __device__ inline long long pcnn_chunk_of(const pcnn_chunking &g, long long sample) {
    if (sample < g.first) return 0;
    const long long r = sample - g.first;
    const long long geo = g.c1 * ((1LL << g.kc) - 1);
    if (r < geo) {
        long long x = r / g.c1 + 1;
        int lg = 0;
        while (x >>= 1) ++lg;
        return 1 + lg;
    }
    return 1 + g.kc + (r - geo) / g.cmax;
}
__host__ __device__ inline long long pcnn_chunk_size(const pcnn_chunking &g, long long k) {
    return k == 0 ? g.first : (k <= g.kc ? g.c1 << (k - 1) : g.cmax);
}
struct pcnn_persist_gate {
    const unsigned *flags;
    unsigned tag;
    pcnn_chunking chunks;
};
// fresh bit 0: start at sample 0 / step 0 (no device-side counter read); bit 1: the error sum restarts at 0
int pcnn_persist_run(pcnn_ctx *ctx, const pcnn_split_binding &s, int B, long nsteps, const pcnn_persist_gate *gate = nullptr,
                     float *step_err_host = nullptr, int fresh = 0, double *done_host = nullptr, unsigned done_tag = 0);
int pcnn_persist_check(pcnn_ctx *ctx);
// comm.cu
int pcnn_comm_allreduce_packed(pcnn_ctx *ctx);
// The opaque plan of include/pcnn.h: what every kernel family's plan holds of its parameters, which pcnn_conv_plan_set_params and
// the optimizer (optim.cu) refresh from fp32 masters in device memory, and the family's forward.  Each family derives from it:
// ToeplitzPlan (conv_tc.cu), ConvWidePlan (conv_wide_tc.cu), LinearPlan (linear_tc.cu), DwConvPlan (dwconv_nhwc.cu) and GConvPlan
// (gconv_nhwc.cu).  pcnn_conv_tc_fwd runs fwd, pcnn_conv_tc_plan_destroy deletes the plan.
//   - w: the bf16 operand, element i of the fp32 master (KRSC, [O][P][Q][C] for a linear plan, [C][R][S] for a depthwise one,
//     [K][R][S][Cg] for a grouped one) at w[(i / cols) * pitch + i % cols], or null for a row-Toeplitz plan, where one filter
//     element feeds V * Qt operand entries (its load_filters gathers them; the optimizer leaves them to pcnn_conv_plan_set_params);
//   - n: the elements of that master; bias: the plan's fp32 copy of the bias ([K]), null for a plan without one.
struct pcnn_conv_plan {
    void *w = nullptr;
    int cols = 0, pitch = 0;
    long long n = 0;
    float *bias = nullptr;
    int K = 0;
    virtual ~pcnn_conv_plan() {
        if (w) cudaFree(w);
        if (bias) cudaFree(bias);
    }
    // y from x with the plan's operand, enqueued on the context's stream (pcnn_conv_tc_fwd has checked the arguments and x's alignment)
    virtual int fwd(pcnn_ctx *ctx, const void *x_bf16, void *y_bf16) = 0;
    // the operand from the fp32 master in device memory, rounded to bf16 on the context's stream; by default the layout of w above
    virtual int load_filters(pcnn_ctx *ctx, const float *filt_dev) {
        return pcnn_f32_to_bf16_rows(ctx, filt_dev, w, (long)(n / cols), cols, pitch);
    }
};
// The tail every create call shares (conv_tc.cu): `bytes` of device memory at *operand (the plan's operand: w, or the Toeplitz
// matrices), the n host filters converted into it by load_filters through a temporary device copy, a synchronisation, and the K
// host bias values copied to plan->bias when bias_host is given.
int pcnn_plan_upload(pcnn_ctx *ctx, pcnn_conv_plan *plan, void **operand, size_t bytes, const float *filt_host, const float *bias_host);
// The plan as family T, or PCNN_ERR_ARG with "fn: the plan was not made by T::made_by" for a plan of any other family
template <class T>
int plan_as(const char *fn, pcnn_conv_plan *plan, T **out) {
    *out = dynamic_cast<T *>(plan);
    PCNN_REQUIRE(*out, PCNN_ERR_ARG, "%s: the plan was not made by %s", fn, T::made_by);
    return PCNN_OK;
}
// the window rules the depthwise and the grouped convolutions share (dwconv_nhwc.cu): N, H, W, C >= 1, 1 <= R, S <= 7, stride 1..4,
// 0 <= pad <= taps - 1 and a window that fits; refused with PCNN_ERR_ARG and a message naming `fn`; P and Q on success
int nhwc_window_check(const char *fn, int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int *P, int *Q);
// The domain and tiling of the wide forward, which its gradients (conv_wide_bwd_tc.cu) share: one rule, refused with
// PCNN_ERR_ARG and a message that names `fn`, the caller's entry point.  conv_wide_pixel_block picks the Pt x Qt = 128 block
// of a P x Q image and returns the blocks per image.
// Tap r of a window padded by pad_h and dilated by dil_h reads x row st * (p + roff[r]) + rph[r] for output row p:
// r * dil_h - pad_h = st * roff[r] + rph[r] with 0 <= rph[r] < st (floor division, so roff[r] < 0 above the image), i.e. phase
// rph[r] of x at box row p0 + roff[r].  Columns the same with sph / soff, dil_w and pad_w.  At pad 0, dilation 1 these are r % st
// and r / st.
struct ConvWideTaps { int rph[7], roff[7], sph[7], soff[7]; };
struct ConvWideShape { int Pt, Qt, nch, stages, tiles, n_pb, n_qb, npad, P, Q; ConvWideTaps taps; };
int conv_wide_shape(const char *fn, int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w, int dil_h,
                    int dil_w, int row_pitch, int image_rows, ConvWideShape *out);
long long conv_wide_pixel_block(int P, int Q, int *Pt, int *Qt);
// pool_nhwc.cu: the partition of the global average pool's reduction over the pixels of an image, which the gate gradient of
// squeeze-and-excitation (se_nhwc.cu) shares so that both sum in one order.  CTA (n, range, slice) of GAP_THREADS threads owns
// pixels [range * per_cta, (range + 1) * per_cta) and channel groups [slice * Gc, (slice + 1) * Gc); thread t keeps group t % Gc of
// the pixels lane, lane + lanes, ... (lane = t / Gc, GAP_ITERS of them), summed from the first; the lanes are then added in lane
// order, and with several ranges the ranges in range order through fp32 slots.  gap_shape is the domain (refused with
// PCNN_ERR_ARG and a message naming `fn`) and the partition, a function of (N, H, W, C) and the row pitch alone.
constexpr int GAP_THREADS = 256;
constexpr int GAP_ITERS = 8;                // pixels per lane
struct GapArgs {
    int HW, C, G;           // pixels per image, channels, channel groups of VEC
    int Gc, slices;         // groups per CTA, channel slices
    int lanes, per_cta, ranges;
    int pitch;              // row pitch of the pooled [N][pitch] rows
    double hw, rhw;         // float(H W), the divisor, and RN(1 / double(float(H W))) for div_rn
};
int gap_shape(const char *fn, int N, int H, int W, int C, int row_pitch, GapArgs *a);
#ifdef __CUDACC__
// The IEEE quotient RN(a / b) for b >= 1 given rb = RN(1 / double(b)), with no out-of-line slow path: __fdiv_rn branches to one
// for extreme exponents, and the call's register convention spills the sums held across it.  In double, a / b of a float a
// neither overflows nor underflows, so two FMA remainder steps give RN_double(a / b) (Markstein: rb correctly rounded, the
// second step starts from a faithful quotient); rounding that to float is RN(a / b) (53 >= 2 * 24 + 2 bits: double rounding is
// innocuous for a quotient).  Zeros, infinities and NaN take a * rb, which keeps the sign of a zero and propagates the rest.
__device__ __forceinline__ float div_rn(float a, double b, double rb) {
    const double ad = a;
    double q = ad * rb;
    q = fma(fma(-b, q, ad), rb, q);
    q = fma(fma(-b, q, ad), rb, q);
    return a == 0.0f || !isfinite(a) ? a * (float)rb : __double2float_rn(q);
}
// E(x) = exp(x) in fp32 as a fixed sequence of round-to-nearest operations with no contraction, so that a numpy float32 replay
// gives the same bits (expf / __expf cannot be replayed).  include/pcnn.h states the sequence and the constants; max error 1.30
// ulp over the finite inputs.  Cody-Waite: k = rint(x log2e); k ln2_hi is exact (15 significant bits times |k| <= 150) and so is
// x - k ln2_hi (Sterbenz); a degree-6 Horner polynomial on |r| <= ln2 / 2; 2^k as two exact powers of two, so that a subnormal
// result is rounded once.  x > 88.7228317 gives +Inf, x < -103.972076 gives +0, NaN gives NaN.
__device__ __forceinline__ float exp_f32(float x) {
    if (x > 88.7228317f) return __int_as_float(0x7f800000);
    if (x < -103.972076f) return 0.0f;
    const float k = rintf(__fmul_rn(x, 1.44269502f));
    const float r = __fsub_rn(__fsub_rn(x, __fmul_rn(k, 0.693145752f)), __fmul_rn(k, 1.42860677e-06f));
    float p = 0.00138436025f;
    p = __fadd_rn(__fmul_rn(p, r), 0.00837419648f);
    p = __fadd_rn(__fmul_rn(p, r), 0.0416680053f);
    p = __fadd_rn(__fmul_rn(p, r), 0.166664302f);
    p = __fadd_rn(__fmul_rn(p, r), 0.49999994f);
    p = __fadd_rn(__fmul_rn(p, r), 1.0f);
    p = __fadd_rn(__fmul_rn(p, r), 1.0f);
    const int ki = __float2int_rn(k), k1 = ki >> 1, k2 = ki - k1;      // a NaN x gives ki = 0 and p = NaN
    return __fmul_rn(__fmul_rn(p, __int_as_float((k1 + 127) << 23)), __int_as_float((k2 + 127) << 23));
}
// log1p(e) for e in (-1, 1], replayable like exp_f32 (include/pcnn.h states the sequence; max error 0.92 ulp).  u = RN(1 + e)
// and its rounding error c = e - (u - 1), which both subtractions give exactly; u = 2^k m with m in [sqrt(1/2), sqrt(2)) from the
// bits, so f = m - 1 is exact; log1p(f) by fdlibm's s = f / (2 + f) series; c / u is the first-order correction for 1 + e != u.
// One function serves both the Box-Muller radius (e = u1 - 1, exact) and the softplus of the logit losses (e = E(-|x|) in [0, 1]).
__device__ __forceinline__ float log1p_f32(float e) {
    const float u = __fadd_rn(1.0f, e);
    const float c = __fsub_rn(e, __fsub_rn(u, 1.0f));
    const int ix = __float_as_int(u) + (0x3F800000 - 0x3F3504F3);
    const float k = (float)((ix >> 23) - 0x7F);
    const float f = __fsub_rn(__int_as_float((ix & 0x7FFFFF) + 0x3F3504F3), 1.0f);
    const float s = __fdiv_rn(f, __fadd_rn(2.0f, f));
    const float z = __fmul_rn(s, s), w = __fmul_rn(z, z);
    const float t1 = __fmul_rn(w, __fadd_rn(__int_as_float(0x3ECCCCE1), __fmul_rn(w, __int_as_float(0x3E789E26))));
    const float t2 = __fmul_rn(z, __fadd_rn(__int_as_float(0x3F2AAAAA), __fmul_rn(w, __int_as_float(0x3E91E9EE))));
    const float hfsq = __fmul_rn(__fmul_rn(0.5f, f), f);
    const float lo = __fadd_rn(__fmul_rn(k, __int_as_float(0x3717F7D1)), __fdiv_rn(c, u));
    const float v = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(s, __fadd_rn(hfsq, __fadd_rn(t2, t1))), lo), hfsq), f);
    return __fadd_rn(v, __fmul_rn(k, __int_as_float(0x3F317180)));
}
// sin and cos of 2 pi k 2^-24 for integer 0 <= k < 2^24, replayable (include/pcnn.h; max error 1.72 ulp).  The octant k >> 21
// and the position in it are exact integers, so the only reduction is a reflection t -> 1 - t in odd octants; then sin(pi t / 4)
// = t S(t^2) and cos(pi t / 4) = C(t^2) on 0 <= t <= 1, and the octant swaps and negates them.
__device__ __forceinline__ void sincos_2pi_f32(unsigned k, float *sn, float *cs) {
    const unsigned o = k >> 21, j = k & 0x1FFFFFu;
    const float t = __fmul_rn((float)((o & 1) ? 0x200000u - j : j), __int_as_float(0x35000000));   // 2^-21
    const float z = __fmul_rn(t, t);
    float p = __int_as_float(0x34A60075);
    p = __fadd_rn(__fmul_rn(p, z), __int_as_float(0xB81965B4));
    p = __fadd_rn(__fmul_rn(p, z), __int_as_float(0x3B2335DE));
    p = __fadd_rn(__fmul_rn(p, z), __int_as_float(0xBDA55DE7));
    p = __fadd_rn(__fmul_rn(p, z), __int_as_float(0x3F490FDB));
    const float S = __fmul_rn(t, p);
    float q = __int_as_float(0xB2D08CC9);
    q = __fadd_rn(__fmul_rn(q, z), __int_as_float(0x3670F449));
    q = __fadd_rn(__fmul_rn(q, z), __int_as_float(0xB9AAE9DE));
    q = __fadd_rn(__fmul_rn(q, z), __int_as_float(0x3C81E0F8));
    q = __fadd_rn(__fmul_rn(q, z), __int_as_float(0xBE9DE9E6));
    const float C = __fadd_rn(__fmul_rn(q, z), 1.0f);
    const bool swap = ((o + 1) >> 1) & 1;                    // octants 1, 2, 5, 6
    const float a = swap ? C : S, b = swap ? S : C;
    *sn = o >= 4 ? -a : a;
    *cs = (o >= 2 && o <= 5) ? -b : b;
}
#endif
// conv_wgrad_tc.cu: dw[o] = sum over i of slots[i][o] for o < nout, in a fixed order (deterministic, no atomics)
int pcnn_conv_wgrad_reduce_slots(pcnn_ctx *ctx, const float *slots, float *dw, int nslots, int nout);
// pcnn_abi.cu: at least `bytes` of device scratch, valid until the next call that asks for more (work using it must be
// enqueued on ctx->stream)
int pcnn_scratch(pcnn_ctx *ctx, size_t bytes, void **out);
