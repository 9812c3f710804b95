// parallel-cnn_b200/csrc/fused_kernels.cu -- the fast tier: one kernel runs forward_pass + makeError +
// vectorNorm + back_pass (Main.cpp:59-144, 167-169) for a whole mini-batch with frozen parameters and
// leaves per-CTA partial packed gradients; a second kernel reduces the partials in a fixed order and applies
// the update.  Nothing but the input image (784 B as u8) and the label crosses HBM per sample; parameters
// (9.4 KB) are read once per CTA and all activations live in registers / shared memory.
//
// Work decomposition (DESIGN.md "fused step kernel"):
//   * CTA = 224 threads = 216 workers + 8 helpers, 2 CTAs per SM; a CTA walks images b = blockIdx.x, +gridDim.x, ...
//   * worker t <-> (feature map m = t / 36, pooling window (wx, wy) = ((t % 36) / 6, t % 6)).  The 4x4 block of
//     c1 outputs feeding one s1 output depends on an 8x8 input patch, so fp_c1 -> sigmoid -> fp_s1 -> sigmoid and
//     the whole c1/s1 backward chain (bp_output_c1, bp_preact_c1, bp_weight_c1, bp_weight_s1, both bias sums)
//     are thread-local: no shared-memory traffic and no synchronisation between those layers.
//   * the only cross-thread step is the 216 -> 10 fully connected layer: warp-shuffle tree + one shared-memory
//     hop (fp_preact_f), then a broadcast of d_preact_f[10] back (bp_output_s1 / bp_weight_f).
//   * weight-gradient accumulators (25 c1 taps, 16 s1 taps, 10 f weights, bias sums) stay in registers across all
//     images of the CTA and are reduced once at the end (warp shuffles + fixed-order shared-memory sums), so the
//     result is deterministic: no atomics anywhere.
//   * images are staged by 1-D TMA bulk copies (cp.async.bulk + mbarrier), double buffered.
//
// Numerics: fp32 with FMA contraction and tree-ordered sums, float sigmoid 1/(1+expf(-v)); differs from the
// reference's sequential un-fused sums and double exp by a few ulp per value (tolerances in tests/ and DESIGN.md).
#include "fused_body.cuh"

using namespace pcnn_fused;

namespace {

struct FusedArgs {
    const void *images;          // [n_total][784] u8 or f32
    const uint8_t *labels;       // [n_total]
    const float *params;         // [NPACK]
    float *slots;                // [gridDim.x][NPACK]      (TRAIN)
    float *f_out;                // [B][10] or null         (EVAL)
    uint8_t *pred;               // [B] or null             (EVAL)
    int *wrong;                  // misclassification counter or null (EVAL)
    const long long *cursor;     // device-side global sample cursor or null
    long long first;             // used when cursor == null
    long long n_total;           // samples in the split (cursor mode clamps the batch at the end)
    int B;                       // per-rank batch
    int rank, world;
};

template <typename InT, bool TRAIN>
__global__ void __launch_bounds__(NT, FUSED_CTAS_PER_SM) k_fused(const FusedArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    FusedSmem<InT> &S = *reinterpret_cast<FusedSmem<InT> *>(smem_raw);
    const ThreadId id;

    // this rank's slice of the (global) batch
    long long base = a.cursor ? *a.cursor : a.first;
    base += (long long)a.rank * a.B;
    const long long avail = a.n_total - base;
    const int nb = avail <= 0 ? 0 : (avail < a.B ? (int)avail : a.B);
    const InT *img_base = reinterpret_cast<const InT *>(a.images) + base * PCNN_IMG;
    const uint8_t *lab_base = a.labels ? a.labels + base : nullptr;

    init_barriers(S);
    const int b0 = blockIdx.x;
    if (id.t == 0) {
        issue_params(S, a.params);
        if (b0 < nb) issue_image(S, 0, img_base + (long long)b0 * PCNN_IMG);
    }
    __syncwarp();   // lane 0 rejoins its warp (see image_pass)
    Acc A;
    A.zero();
    int li = 0;
    for (int b = b0; b < nb; b += gridDim.x, ++li) {
        const int bn = b + gridDim.x;
        EvalOut ev;
        ev.f_out = (!TRAIN && a.f_out) ? a.f_out + (long long)b * PCNN_F : nullptr;
        ev.pred = (!TRAIN && a.pred) ? a.pred + b : nullptr;
        ev.has_label = lab_base != nullptr;
        image_pass<InT, TRAIN>(S, id, li, lab_base ? lab_base + b : nullptr,
                               bn < nb ? img_base + (long long)bn * PCNN_IMG : nullptr, li == 0 ? 0 : -1, A, ev);
    }
    if (!TRAIN) {
        if (id.t == 0 && a.wrong && A.wrong) atomicAdd(a.wrong, A.wrong);
        if (li == 0) mbar_wait(&S.mbar[2], 0);   // never exit with the parameter copy still in flight
        return;
    }
    if (li == 0) mbar_wait(&S.mbar[2], 0);
    cta_epilogue(S, id, A, FloatSink{a.slots + (long long)blockIdx.x * NPACK});
}
// ---- second kernel: fixed-order reduction of the per-CTA slots, optional update ------------------------------
// block = 256 threads = 32 packed entries x 8 slot-phases; entry p of the packed vector is summed over slots
// phase, phase+8, ... by each phase and the 8 partials are added in phase order.
struct ReduceArgs {
    const float *slots;
    int nslots;
    float *grads;               // [NPACK] out
    float *params;              // [NPACK] in/out (when update)
    double *err_total;          // running error-norm sum
    float *step_err;            // optional ring of per-step error sums, indexed by *step_idx
    const int *step_idx;
    const long long *cursor_in; // cursor mode: read to compute the effective global batch
    long long n_total;
    int B, world, rank_local;
    float dt;
    int update;                 // 1: apply update here (single GPU); 0: leave grads for the all-reduce
};

__global__ void __launch_bounds__(256) k_reduce_slots(const ReduceArgs a) {
    __shared__ float part[8][33];
    const int pl = threadIdx.x & 31, phase = threadIdx.x >> 5;
    const int p = blockIdx.x * 32 + pl;
    float s = 0.0f;
    if (p < NPACK)
        for (int k = phase; k < a.nslots; k += 8) s += a.slots[(long long)k * NPACK + p];
    part[phase][pl] = s;
    __syncthreads();
    if (phase == 0 && p < NPACK) {
        float g = part[0][pl];
#pragma unroll
        for (int q = 1; q < 8; ++q) g += part[q][pl];
        a.grads[p] = g;
        if (a.update) {
            if (p < NPARAM) {
                const float step = a.dt / (float)effective_global_batch(a.cursor_in ? *a.cursor_in : 0, a.cursor_in != nullptr,
                                                                        a.n_total, a.B, a.world, a.rank_local);
                a.params[p] = updated_entry(a.params[p], p, g, step);
            } else {
                *a.err_total += (double)g;
                if (a.step_err) a.step_err[*a.step_idx & (STEP_ERR_CAP - 1)] = g;
            }
        }
    }
}

// cursor advance must not race with the reads above -> its own tiny kernel at the end of the step
__global__ void k_advance_cursor(long long *cursor, long long n_total, long long stride, int *step_idx) {
    long long c = *cursor + stride;
    if (c >= n_total) c = 0;
    *cursor = c;
    *step_idx += 1;
}

// update after an all-reduce (grads already hold the global sum)
struct UpdateArgs {
    const float *grads;
    float *params;
    double *err_total;
    float *step_err;
    const int *step_idx;
    const long long *cursor_in;
    long long n_total;
    int B, world, rank_local;
    float dt;
};
__global__ void __launch_bounds__(256) k_update(const UpdateArgs a) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= NPACK) return;
    const float g = a.grads[p];
    if (p < NPARAM) {
        const float step = a.dt / (float)effective_global_batch(a.cursor_in ? *a.cursor_in : 0, a.cursor_in != nullptr, a.n_total,
                                                                a.B, a.world, a.rank_local);
        a.params[p] = updated_entry(a.params[p], p, g, step);
    } else {
        *a.err_total += (double)g;
        if (a.step_err) a.step_err[*a.step_idx & (STEP_ERR_CAP - 1)] = g;
    }
}

template <typename InT, bool TRAIN> int configure_fused() {
    cudaError_t e = cudaFuncSetAttribute(k_fused<InT, TRAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)sizeof(FusedSmem<InT>));
    if (e != cudaSuccess) return pcnn_fail_cuda(e, "cudaFuncSetAttribute(k_fused)", __FILE__, __LINE__);
    return PCNN_OK;
}

int fused_grid(pcnn_ctx *ctx, int B) {
    int cap = ctx->sm_count * FUSED_CTAS_PER_SM;
    if (cap > MAX_SLOTS) cap = MAX_SLOTS;
    return B < cap ? B : cap;
}

template <bool TRAIN> int launch_fused(pcnn_ctx *ctx, const FusedArgs &a, int pixel_type, int grid) {
    if (pixel_type == PCNN_U8)
        k_fused<uint8_t, TRAIN><<<grid, NT, sizeof(FusedSmem<uint8_t>), ctx->stream>>>(a);
    else
        k_fused<float, TRAIN><<<grid, NT, sizeof(FusedSmem<float>), ctx->stream>>>(a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------ internal launchers
// called once per context (pcnn_create): opt the four instantiations into their dynamic shared-memory size
int pcnn_fused_configure() {
    int rc;
    if ((rc = configure_fused<uint8_t, true>())) return rc;
    if ((rc = configure_fused<uint8_t, false>())) return rc;
    if ((rc = configure_fused<float, true>())) return rc;
    if ((rc = configure_fused<float, false>())) return rc;
    return PCNN_OK;
}

int pcnn_launch_fused_grad(pcnn_ctx *ctx, const pcnn_step_src &src, int B, int *grid_out) {
    FusedArgs a{};
    a.images = src.images;
    a.labels = src.labels;
    a.params = ctx->d_params;
    a.slots = ctx->d_slots;
    a.cursor = src.use_cursor ? ctx->d_cursor : nullptr;
    a.first = src.first;
    a.n_total = src.n_total;
    a.B = B;
    a.rank = (src.use_cursor && !src.rank_local) ? ctx->rank : 0;
    a.world = ctx->world;
    int grid = fused_grid(ctx, B);
    if (grid_out) *grid_out = grid;
    return launch_fused<true>(ctx, a, src.pixel_type, grid);
}

int pcnn_launch_reduce(pcnn_ctx *ctx, int grid_slots, int B, const pcnn_step_src &src, bool update, bool record_err) {
    ReduceArgs r{};
    r.slots = ctx->d_slots;
    r.nslots = grid_slots;
    r.grads = ctx->d_grads;
    r.params = ctx->d_params;
    r.err_total = ctx->d_err_total;
    r.step_err = record_err ? ctx->d_step_err : nullptr;
    r.step_idx = ctx->d_step_idx;
    r.cursor_in = src.use_cursor ? ctx->d_cursor : nullptr;
    r.n_total = src.n_total;
    r.B = B;
    r.world = ctx->world;
    r.rank_local = src.rank_local ? 1 : 0;
    r.dt = ctx->lr;
    r.update = update ? 1 : 0;
    k_reduce_slots<<<(NPACK + 31) / 32, 256, 0, ctx->stream>>>(r);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

int pcnn_launch_update(pcnn_ctx *ctx, int B, const pcnn_step_src &src, bool record_err) {
    UpdateArgs u{};
    u.grads = ctx->d_grads;
    u.params = ctx->d_params;
    u.err_total = ctx->d_err_total;
    u.step_err = record_err ? ctx->d_step_err : nullptr;
    u.step_idx = ctx->d_step_idx;
    u.cursor_in = src.use_cursor ? ctx->d_cursor : nullptr;
    u.n_total = src.n_total;
    u.B = B;
    u.world = ctx->world;
    u.rank_local = src.rank_local ? 1 : 0;
    u.dt = ctx->lr;
    k_update<<<(NPACK + 255) / 256, 256, 0, ctx->stream>>>(u);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

static int launch_advance(pcnn_ctx *ctx, const pcnn_step_src &src, int B) {
    const long long stride = src.rank_local ? (long long)B : (long long)B * ctx->world;
    k_advance_cursor<<<1, 1, 0, ctx->stream>>>(ctx->d_cursor, src.n_total, stride, ctx->d_step_idx);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

// one full step on the context's stream: gradient kernel, slot reduction, [all-reduce + update], [cursor advance]
static int enqueue_step(pcnn_ctx *ctx, const pcnn_step_src &src, int B) {
    int grid = 0, rc;
    // peers attached without NCCL: only the persistent kernel can exchange the gradient; a per-step kernel chain would
    // update every replica with its LOCAL gradient at 1/world of the step size
    PCNN_REQUIRE(ctx->world == 1 || ctx->nccl_comm, PCNN_ERR_STATE,
                 "single-step entry points need pcnn_comm_init_rank when world > 1 (peer attach serves pcnn_train_steps / pcnn_learn only)");
    if ((rc = pcnn_launch_fused_grad(ctx, src, B, &grid))) return rc;
    const bool distributed = ctx->world > 1 && ctx->nccl_comm;
    if ((rc = pcnn_launch_reduce(ctx, grid, B, src, !distributed, src.use_cursor && !distributed))) return rc;
    if (distributed) {
        if ((rc = pcnn_comm_allreduce_packed(ctx))) return rc;
        if ((rc = pcnn_launch_update(ctx, B, src, src.use_cursor))) return rc;
    }
    if (src.use_cursor && (rc = launch_advance(ctx, src, B))) return rc;
    return PCNN_OK;
}

static pcnn_step_src src_of(const pcnn_split_binding &s, long first, bool use_cursor) {
    pcnn_step_src r;
    r.images = s.images;
    r.labels = s.labels;
    r.pixel_type = s.pixel_type;
    r.n_total = s.n;
    r.first = first;
    r.use_cursor = use_cursor;
    r.rank_local = s.rank_local;
    return r;
}
static pcnn_step_src src_of_buffers(const void *images, int pixel_type, const uint8_t *labels, int B) {
    pcnn_step_src r;
    r.images = images;
    r.labels = labels;
    r.pixel_type = pixel_type;
    r.n_total = B;
    r.first = 0;
    r.use_cursor = false;
    r.rank_local = true;
    return r;
}

static int check_batch_args(pcnn_ctx *ctx, const char *fn, const void *images, int pixel_type, const uint8_t *labels, int B) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "%s: ctx is NULL", fn);
    PCNN_REQUIRE(images && labels, PCNN_ERR_ARG, "%s: NULL images/labels", fn);
    PCNN_REQUIRE(pixel_type == PCNN_U8 || pixel_type == PCNN_F32, PCNN_ERR_ARG, "%s: bad pixel type %d", fn, pixel_type);
    PCNN_REQUIRE(B > 0, PCNN_ERR_ARG, "%s: batch must be positive (got %d)", fn, B);
    PCNN_REQUIRE(((uintptr_t)images & 15) == 0, PCNN_ERR_ARG, "%s: images must be 16-byte aligned (bulk-copy source)", fn);
    return PCNN_OK;
}

// ------------------------------------------------------------------------------------------ C ABI: training
extern "C" int pcnn_compute_grads(pcnn_ctx *ctx, const void *dev_images, int pixel_type, const uint8_t *dev_labels, int B) {
    int rc = check_batch_args(ctx, "pcnn_compute_grads", dev_images, pixel_type, dev_labels, B);
    if (rc) return rc;
    pcnn_device_guard g(ctx->device);
    int grid = 0;
    const pcnn_step_src src = src_of_buffers(dev_images, pixel_type, dev_labels, B);
    if ((rc = pcnn_launch_fused_grad(ctx, src, B, &grid))) return rc;
    return pcnn_launch_reduce(ctx, grid, B, src, false, false);   // reduce only: no update, err_total untouched
}

extern "C" int pcnn_train_step_dev(pcnn_ctx *ctx, const void *dev_images, int pixel_type, const uint8_t *dev_labels, int B) {
    int rc = check_batch_args(ctx, "pcnn_train_step_dev", dev_images, pixel_type, dev_labels, B);
    if (rc) return rc;
    pcnn_device_guard g(ctx->device);
    return enqueue_step(ctx, src_of_buffers(dev_images, pixel_type, dev_labels, B), B);
}

extern "C" int pcnn_train_step(pcnn_ctx *ctx, long first, int B) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_train_step: ctx is NULL");
    const pcnn_split_binding &s = ctx->split[PCNN_TRAIN_SET];
    PCNN_REQUIRE(s.n > 0, PCNN_ERR_STATE, "pcnn_train_step: no training split bound (pcnn_dataset_upload/bind)");
    PCNN_REQUIRE(B > 0 && first >= 0 && first + (long)B <= s.n, PCNN_ERR_ARG,
                 "pcnn_train_step: samples [%ld, %ld) outside the split of %ld", first, first + (long)B, s.n);
    pcnn_device_guard g(ctx->device);
    return enqueue_step(ctx, src_of(s, first, false), B);
}

// Cursor-driven steps are replayed from CUDA graphs.  A run of nsteps is decomposed into graphs of 1024 / 256 / 64 /
// 16 / 4 / 1 steps; the sample position and the step-error slot come from device-side counters, so one graph per
// (size, B, split) serves any position.
static const int GRAPH_SIZES[] = {1024, 256, 64, 16, 4, 1};

static int get_step_graph(pcnn_ctx *ctx, const pcnn_split_binding &s, int B, int nsteps, cudaGraphExec_t *out) {
    pcnn_graph_key key{B, nsteps, ctx->world, s.pixel_type, s.rank_local ? 1 : 0, s.images, s.labels, s.n};
    auto it = ctx->graphs.find(key);
    if (it != ctx->graphs.end()) { *out = it->second; return PCNN_OK; }
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    PCNN_CUDA(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
    int rc = PCNN_OK;
    const long before = ctx->launches;
    const pcnn_step_src src = src_of(s, 0, true);
    for (int k = 0; k < nsteps && rc == PCNN_OK; ++k) rc = enqueue_step(ctx, src, B);
    cudaError_t e = cudaStreamEndCapture(ctx->stream, &graph);
    ctx->launches = before;   // captured, not launched
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (e != cudaSuccess) return pcnn_fail_cuda(e, "cudaStreamEndCapture", __FILE__, __LINE__);
    e = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) return pcnn_fail_cuda(e, "cudaGraphInstantiate", __FILE__, __LINE__);
    ctx->graphs[key] = exec;
    *out = exec;
    return PCNN_OK;
}

static bool use_persistent(pcnn_ctx *ctx) {
    const bool can = ctx->persist_cap > 0 && (ctx->world == 1 || ctx->p2p_ready);
    if (ctx->step_mode == PCNN_MODE_GRAPH) return false;
    return can;   // AUTO and PERSISTENT: whenever the persistent kernel can serve the configuration
}

static int run_cursor_steps(pcnn_ctx *ctx, const pcnn_split_binding &s, int B, long nsteps, bool launch) {
    if (ctx->step_mode == PCNN_MODE_PERSISTENT)
        PCNN_REQUIRE(use_persistent(ctx), PCNN_ERR_STATE, "persistent mode requested but peers are not attached");
    if (use_persistent(ctx)) return launch ? pcnn_persist_run(ctx, s, B, nsteps) : PCNN_OK;
    PCNN_REQUIRE(ctx->world == 1 || ctx->nccl_comm, PCNN_ERR_STATE,
                 "distributed steps need pcnn_comm_init_rank (graph mode) or pcnn_p2p_attach (persistent mode)");
    const bool distributed = ctx->world > 1 && ctx->nccl_comm;
    for (int size : GRAPH_SIZES) {
        while (nsteps >= size) {
            cudaGraphExec_t exec = nullptr;
            int rc = get_step_graph(ctx, s, B, size, &exec);
            if (rc) return rc;
            if (!launch) { nsteps %= size; break; }     // prepare mode: instantiate each size once
            PCNN_CUDA(cudaGraphLaunch(exec, ctx->stream));
            ctx->launches += (long)size * (distributed ? 4 : 3);   // our kernels per step (the NCCL kernel is not ours)
            nsteps -= size;
        }
    }
    return PCNN_OK;
}

static int set_cursor(pcnn_ctx *ctx, long long v) {
    // pinned scratch so the copy is asynchronous; synchronise first so h_scalar is not overwritten while in flight
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    *reinterpret_cast<long long *>(ctx->h_scalar) = v;
    PCNN_CUDA(cudaMemcpyAsync(ctx->d_cursor, ctx->h_scalar, sizeof(long long), cudaMemcpyHostToDevice, ctx->stream));
    return PCNN_OK;
}

extern "C" int pcnn_train_steps(pcnn_ctx *ctx, long first, int B, int nsteps) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_train_steps: ctx is NULL");
    const pcnn_split_binding &s = ctx->split[PCNN_TRAIN_SET];
    PCNN_REQUIRE(s.n > 0, PCNN_ERR_STATE, "pcnn_train_steps: no training split bound");
    PCNN_REQUIRE(B > 0 && nsteps > 0 && first >= -1 && first < s.n, PCNN_ERR_ARG, "pcnn_train_steps: bad arguments");
    pcnn_device_guard g(ctx->device);
    int rc;
    if (first >= 0 && (rc = set_cursor(ctx, first))) return rc;     // first == -1: continue at the device cursor
    return run_cursor_steps(ctx, s, B, nsteps, true);
}

extern "C" int pcnn_train_steps_prepare(pcnn_ctx *ctx, int B, int nsteps) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_train_steps_prepare: ctx is NULL");
    const pcnn_split_binding &s = ctx->split[PCNN_TRAIN_SET];
    PCNN_REQUIRE(s.n > 0, PCNN_ERR_STATE, "pcnn_train_steps_prepare: no training split bound");
    PCNN_REQUIRE(B > 0 && nsteps > 0, PCNN_ERR_ARG, "pcnn_train_steps_prepare: bad arguments");
    pcnn_device_guard g(ctx->device);
    return run_cursor_steps(ctx, s, B, nsteps, false);
}

extern "C" int pcnn_learn(pcnn_ctx *ctx, int B, int epochs, float *mean_err_out) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_learn: ctx is NULL");
    const pcnn_split_binding &s = ctx->split[PCNN_TRAIN_SET];
    PCNN_REQUIRE(s.n > 0, PCNN_ERR_STATE, "pcnn_learn: no training split bound");
    PCNN_REQUIRE(B > 0 && epochs > 0, PCNN_ERR_ARG, "pcnn_learn: bad arguments");
    pcnn_device_guard g(ctx->device);
    const long gb = (long)B * ctx->world;
    const long steps_per_epoch = (s.n + gb - 1) / gb;
    int rc;
    double err = 0.0;
    for (int ep = 0; ep < epochs; ++ep) {
        if ((rc = set_cursor(ctx, 0))) return rc;
        if ((rc = pcnn_err_sum(ctx, nullptr, 1))) return rc;
        if ((rc = run_cursor_steps(ctx, s, B, steps_per_epoch, true))) return rc;
        if ((rc = pcnn_err_sum(ctx, &err, 0))) return rc;
    }
    if (mean_err_out) *mean_err_out = (float)(err / (double)s.n);
    return PCNN_OK;
}

// ------------------------------------------------------------------------------------------ host-buffer entry points
static int ensure_stage(pcnn_ctx *ctx, long samples) {
    if (samples <= ctx->stage_cap_samples) return PCNN_OK;
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    PCNN_CUDA(cudaStreamSynchronize(ctx->copy_stream));
    pcnn_drop_graphs(ctx);                                   // cached graphs bake the staging pointers in
    for (int i = 0; i < 2; ++i) {
        if (ctx->h_stage[i]) cudaFreeHost(ctx->h_stage[i]);
        if (ctx->d_stage[i]) cudaFree(ctx->d_stage[i]);
        if (ctx->h_stage_lab[i]) cudaFreeHost(ctx->h_stage_lab[i]);
        if (ctx->d_stage_lab[i]) cudaFree(ctx->d_stage_lab[i]);
        size_t bytes = (size_t)samples * PCNN_IMG * sizeof(float);   // sized for the larger pixel type
        PCNN_CUDA(cudaMallocHost(&ctx->h_stage[i], bytes));
        PCNN_CUDA(cudaMalloc(&ctx->d_stage[i], bytes));
        PCNN_CUDA(cudaMallocHost((void **)&ctx->h_stage_lab[i], (size_t)samples));
        PCNN_CUDA(cudaMalloc((void **)&ctx->d_stage_lab[i], (size_t)samples));
    }
    ctx->stage_cap_samples = samples;
    return PCNN_OK;
}

extern "C" int pcnn_train_step_host(pcnn_ctx *ctx, const void *host_images, int pixel_type, const uint8_t *host_labels,
                                    int B, float *err_sum_out) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_train_step_host: ctx is NULL");
    PCNN_REQUIRE(host_images && host_labels && B > 0, PCNN_ERR_ARG, "pcnn_train_step_host: NULL buffers or B <= 0");
    PCNN_REQUIRE(pixel_type == PCNN_U8 || pixel_type == PCNN_F32, PCNN_ERR_ARG, "pcnn_train_step_host: bad pixel type");
    pcnn_device_guard g(ctx->device);
    int rc;
    if ((rc = ensure_stage(ctx, B))) return rc;
    const size_t ib = (size_t)B * PCNN_IMG * (pixel_type == PCNN_F32 ? 4 : 1);
    // the caller's buffers may be pageable: the copies below stage through the driver if so, pinned memory
    // (cudaHostRegister'ed or cudaMallocHost'ed by the caller) goes by DMA directly
    PCNN_CUDA(cudaMemcpyAsync(ctx->d_stage[0], host_images, ib, cudaMemcpyHostToDevice, ctx->stream));
    PCNN_CUDA(cudaMemcpyAsync(ctx->d_stage_lab[0], host_labels, (size_t)B, cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = enqueue_step(ctx, src_of_buffers(ctx->d_stage[0], pixel_type, ctx->d_stage_lab[0], B), B))) return rc;
    // the step's error sum is element OFF_ERR of the packed gradient (all-reduced when distributed)
    PCNN_CUDA(cudaMemcpyAsync(ctx->h_scalar, ctx->d_grads + OFF_ERR, sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    if (err_sum_out) *err_sum_out = *ctx->h_scalar;
    return PCNN_OK;
}

// Graph / NCCL mode: learn() over a HOST dataset: chunks of `chunk_steps` batches are copied on the copy stream into one of two
// device staging buffers while the compute stream trains on the other; per-step error sums are read back.
static int learn_host_chunked(pcnn_ctx *ctx, const void *host_images, int pixel_type, const uint8_t *host_labels,
                              long n, int B, int epochs, float *mean_err_out) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_learn_host: ctx is NULL");
    PCNN_REQUIRE(host_images && host_labels && n > 0 && B > 0 && epochs > 0, PCNN_ERR_ARG, "pcnn_learn_host: bad arguments");
    PCNN_REQUIRE(pixel_type == PCNN_U8 || pixel_type == PCNN_F32, PCNN_ERR_ARG, "pcnn_learn_host: bad pixel type");
    pcnn_device_guard g(ctx->device);
    const size_t px = (pixel_type == PCNN_F32 ? 4 : 1);
    // Chunks of ~16 MiB (80 steps at B = 256 u8): the per-chunk fixed cost (two copies, two memsets, events, one launch, one
    // read-back) is then small next to the chunk's compute; the first chunk is ~2 MiB so that the copy nothing
    // can overlap with stays short.
    long chunk_samples = ((long)(16 << 20) / (long)(PCNN_IMG * px));
    chunk_samples = (chunk_samples / B) * B;
    if (chunk_samples < B) chunk_samples = B;
    if (chunk_samples / B > STEP_ERR_CAP) chunk_samples = (long)STEP_ERR_CAP * B;
    long first_chunk = ((long)(2 << 20) / (long)(PCNN_IMG * px) / B) * B;
    if (first_chunk < B) first_chunk = B;
    if (first_chunk > chunk_samples) first_chunk = chunk_samples;
    // data parallel: `host_images` is THIS rank's shard (all ranks must pass equally sized shards); every step
    // all-reduces the packed gradient and divides the step by B * world
    int rc;
    if ((rc = ensure_stage(ctx, chunk_samples))) return rc;
    const char *hi = reinterpret_cast<const char *>(host_images);
    double err = 0.0;
    const long total_steps = (n + B - 1) / B;
    if (total_steps > ctx->h_step_err_cap) {
        PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
        if (ctx->h_step_err) cudaFreeHost(ctx->h_step_err);
        ctx->h_step_err = nullptr;
        PCNN_CUDA(cudaMallocHost((void **)&ctx->h_step_err, (size_t)total_steps * sizeof(float)));
        ctx->h_step_err_cap = total_steps;
    }
    for (int ep = 0; ep < epochs; ++ep) {
        if ((rc = pcnn_err_sum(ctx, nullptr, 1))) return rc;
        int slot = 0;
        long steps_done = 0;
        for (long off = 0, cs = 0; off < n; off += cs, slot ^= 1) {
            const long want = off == 0 ? first_chunk : chunk_samples;
            cs = (n - off < want) ? n - off : want;
            // wait until the compute stream has finished with this staging buffer, then copy into it
            PCNN_CUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_done[slot], 0));
            PCNN_CUDA(cudaMemcpyAsync(ctx->d_stage[slot], hi + (size_t)off * PCNN_IMG * px, (size_t)cs * PCNN_IMG * px,
                                      cudaMemcpyHostToDevice, ctx->copy_stream));
            PCNN_CUDA(cudaMemcpyAsync(ctx->d_stage_lab[slot], host_labels + off, (size_t)cs, cudaMemcpyHostToDevice, ctx->copy_stream));
            PCNN_CUDA(cudaEventRecord(ctx->ev_copy[slot], ctx->copy_stream));
            PCNN_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_copy[slot], 0));
            // train on the chunk: cursor-driven steps over the staging buffer treated as a split of cs samples
            pcnn_split_binding tmp;
            tmp.images = ctx->d_stage[slot];
            tmp.labels = ctx->d_stage_lab[slot];
            tmp.pixel_type = pixel_type;
            tmp.n = cs;
            tmp.rank_local = true;
            PCNN_CUDA(cudaMemsetAsync(ctx->d_cursor, 0, sizeof(long long), ctx->stream));
            PCNN_CUDA(cudaMemsetAsync(ctx->d_step_idx, 0, sizeof(int), ctx->stream));
            const int steps = (int)((cs + B - 1) / B);
            if ((rc = run_cursor_steps(ctx, tmp, B, steps, true))) return rc;
            // every step's result (its error-norm sum) goes back to the host
            PCNN_CUDA(cudaMemcpyAsync(ctx->h_step_err + steps_done, ctx->d_step_err, (size_t)steps * sizeof(float),
                                      cudaMemcpyDeviceToHost, ctx->stream));
            steps_done += steps;
            PCNN_CUDA(cudaEventRecord(ctx->ev_done[slot], ctx->stream));
        }
        if ((rc = pcnn_err_sum(ctx, &err, 0))) return rc;     // blocking read-back of the epoch's error sum
        ctx->step_err_count = steps_done;
    }
    if (mean_err_out) *mean_err_out = (float)(err / ((double)n * ctx->world));   // err is the all-reduced sum
    return PCNN_OK;
}

// Persistent mode: ONE cooperative launch per epoch.  The epoch's samples are staged in HBM chunk by chunk on the copy
// stream (80 GB of HBM: the whole host dataset fits, up to HS_SEGMENT_BYTES per launch); every chunk is followed by a
// 4-byte flag copy, and the kernel -- launched right after the FIRST chunk has been enqueued -- waits on the flag of a
// sample's chunk before it issues that sample's bulk copy.  Per-step error sums go straight to mapped pinned host memory.
// Host work per call: one launch, 2 copies per chunk, one blocking read-back at the end; no per-chunk synchronisation.
static const size_t HS_SEGMENT_BYTES = (size_t)8 << 30;

static int ensure_host_stream(pcnn_ctx *ctx, size_t image_bytes, long labels, long chunks) {
    if (image_bytes <= ctx->hs_image_bytes && labels <= ctx->hs_label_cap && chunks <= ctx->hs_ready_cap) return PCNN_OK;
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    PCNN_CUDA(cudaStreamSynchronize(ctx->copy_stream));
    if (image_bytes > ctx->hs_image_bytes) {
        if (ctx->d_hs_images) cudaFree(ctx->d_hs_images);
        ctx->d_hs_images = nullptr;
        ctx->hs_image_bytes = 0;
        PCNN_CUDA(cudaMalloc(&ctx->d_hs_images, image_bytes));
        ctx->hs_image_bytes = image_bytes;
    }
    if (labels > ctx->hs_label_cap) {
        if (ctx->d_hs_labels) cudaFree(ctx->d_hs_labels);
        ctx->d_hs_labels = nullptr;
        ctx->hs_label_cap = 0;
        PCNN_CUDA(cudaMalloc((void **)&ctx->d_hs_labels, (size_t)labels));
        ctx->hs_label_cap = labels;
    }
    if (chunks > ctx->hs_ready_cap) {
        if (ctx->d_hs_ready) cudaFree(ctx->d_hs_ready);
        ctx->d_hs_ready = nullptr;
        ctx->hs_ready_cap = 0;
        const long cap = chunks < 256 ? 256 : chunks;
        PCNN_CUDA(cudaMalloc((void **)&ctx->d_hs_ready, (size_t)cap * sizeof(unsigned)));
        PCNN_CUDA(cudaMemset(ctx->d_hs_ready, 0, (size_t)cap * sizeof(unsigned)));
        ctx->hs_ready_cap = cap;
    }
    if (!ctx->h_hs_tag) PCNN_CUDA(cudaMallocHost((void **)&ctx->h_hs_tag, sizeof(unsigned)));
    if (!ctx->h_hs_done) {
        PCNN_CUDA(cudaMallocHost((void **)&ctx->h_hs_done, 2 * sizeof(double)));
        ctx->h_hs_done[0] = ctx->h_hs_done[1] = 0.0;
    }
    return PCNN_OK;
}

// pinned per-step result buffer (the kernel writes every step's error sum straight into it)
static int ensure_step_err_host(pcnn_ctx *ctx, long total_steps) {
    if (total_steps <= ctx->h_step_err_cap) return PCNN_OK;
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    if (ctx->h_step_err) cudaFreeHost(ctx->h_step_err);
    ctx->h_step_err = nullptr;
    ctx->h_step_err_cap = 0;
    PCNN_CUDA(cudaMallocHost((void **)&ctx->h_step_err, (size_t)total_steps * sizeof(float)));
    ctx->h_step_err_cap = total_steps;
    return PCNN_OK;
}

// Results (per-step sums, total, completion tag) arrive in pinned host memory straight from the kernel: poll the tag instead of
// paying a stream synchronisation; the stream is queried now and then so that an aborted or failed launch cannot hang the host.
static int wait_done_tag(pcnn_ctx *ctx, unsigned done_tag) {
    volatile unsigned *tagp = reinterpret_cast<volatile unsigned *>(ctx->h_hs_done + 1);
    bool seen = false;
    for (unsigned long spins = 0;; ++spins) {
        if (*tagp == done_tag) { seen = true; break; }
        if ((spins & 4095) == 4095) {
            const cudaError_t q = cudaStreamQuery(ctx->stream);
            if (q == cudaSuccess) { seen = (*tagp == done_tag); break; }
            if (q != cudaErrorNotReady) return pcnn_fail_cuda(q, "persistent training kernel", __FILE__, __LINE__);
        }
    }
    if (!seen) {
        PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
        int rc;
        if ((rc = pcnn_persist_check(ctx))) return rc;
        PCNN_REQUIRE(*tagp == done_tag, PCNN_ERR_STATE, "pcnn_learn_host: the training kernel ended without reporting completion");
    }
    return PCNN_OK;
}

// Page-locked, device-mapped host images (cudaHostAlloc / cudaHostRegister; torch pin_memory): NO staging copy at all.  The
// training kernel's own bulk copies (cp.async.bulk, one 784-pixel image per CTA and step, issued a step ahead) read the pinned
// buffer across PCIe through its device alias, so a step's pixels cross the link exactly once, when a CTA asks for them, and
// the host enqueues one label copy and one launch per epoch -- no chunks, no flags, no copy-engine work to interleave.
static int learn_host_pull(pcnn_ctx *ctx, const void *images_alias, int pixel_type, const uint8_t *host_labels, long n, int B, int epochs,
                           float *mean_err_out) {
    int rc;
    if ((rc = ensure_host_stream(ctx, 0, n, 0))) return rc;
    const long steps = (n + B - 1) / B;
    if ((rc = ensure_step_err_host(ctx, steps))) return rc;
    PCNN_CUDA(cudaMemcpyAsync(ctx->d_hs_labels, host_labels, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));   // 1 byte per image
    pcnn_split_binding tmp;
    tmp.images = images_alias;
    tmp.host_resident = true;
    tmp.labels = ctx->d_hs_labels;
    tmp.pixel_type = pixel_type;
    tmp.n = n;
    tmp.rank_local = true;
    for (int ep = 0; ep < epochs; ++ep) {
        const bool last = ep + 1 == epochs;
        unsigned done_tag = 0;
        if (last) {
            done_tag = ++ctx->hs_serial;
            if (done_tag == 0) done_tag = ++ctx->hs_serial;
        }
        if ((rc = pcnn_persist_run(ctx, tmp, B, steps, nullptr, ctx->h_step_err, 3, last ? ctx->h_hs_done : nullptr, done_tag))) return rc;
        if (last && (rc = wait_done_tag(ctx, done_tag))) return rc;
    }
    ctx->step_err_count = steps;
    if (mean_err_out) *mean_err_out = (float)(ctx->h_hs_done[0] / ((double)n * ctx->world));   // the all-reduced sum of the last epoch
    return PCNN_OK;
}

static int learn_host_streamed(pcnn_ctx *ctx, const void *host_images, int pixel_type, const uint8_t *host_labels, long n, int B,
                               int epochs, float *mean_err_out) {
    const size_t px = (pixel_type == PCNN_F32 ? 4 : 1);
    const size_t img_bytes = (size_t)PCNN_IMG * px;
    // segment = what one launch trains on; a multiple of B so that only the last segment has a tail batch
    long seg_samples = (long)(HS_SEGMENT_BYTES / img_bytes);
    seg_samples = (seg_samples / B) * B;
    if (seg_samples < B) seg_samples = B;
    if (seg_samples > n) seg_samples = n;
    // chunk 0: one batch (at least ~128 KB), then chunks doubling from ~256 KB up to 16 MB (pcnn_chunking)
    pcnn_chunking ch;
    ch.first = (long)((128 << 10) / img_bytes);
    ch.first = ((ch.first + B - 1) / B) * B;
    if (ch.first > seg_samples) ch.first = seg_samples;
    ch.c1 = (long)((256 << 10) / img_bytes);
    if (ch.c1 < 1) ch.c1 = 1;
    ch.cmax = (long)(((size_t)16 << 20) / img_bytes);
    if (ch.cmax < ch.c1) ch.cmax = ch.c1;
    ch.kc = 0;
    while ((ch.c1 << ch.kc) < ch.cmax && ch.kc < 16) ++ch.kc;          // sizes c1, 2 c1, ... < cmax, then cmax
    const long max_chunks = (long)pcnn_chunk_of(ch, seg_samples > 0 ? seg_samples - 1 : 0) + 1;
    int rc;
    if ((rc = ensure_host_stream(ctx, (size_t)seg_samples * img_bytes, seg_samples, max_chunks))) return rc;
    if ((rc = ensure_step_err_host(ctx, (n + B - 1) / B))) return rc;
    const char *hi = reinterpret_cast<const char *>(host_images);
    const bool resident_after_first = seg_samples >= n;      // later epochs re-use the staged copy
    double err = 0.0;
    for (int ep = 0; ep < epochs; ++ep) {
        long steps_done = 0;
        for (long off = 0; off < n; off += seg_samples) {
            const long sn = n - off < seg_samples ? n - off : seg_samples;
            pcnn_split_binding tmp;
            tmp.images = ctx->d_hs_images;
            tmp.labels = ctx->d_hs_labels;
            tmp.pixel_type = pixel_type;
            tmp.n = sn;
            tmp.rank_local = true;
            const long steps = (sn + B - 1) / B;
            const int fresh = 1 | (off == 0 ? 2 : 0);
            const bool last = off + sn >= n && ep + 1 == epochs;        // the launch whose completion ends the call
            unsigned done_tag = 0;
            if (last) {
                done_tag = ++ctx->hs_serial;
                if (done_tag == 0) done_tag = ++ctx->hs_serial;
            }
            if (ep > 0 && resident_after_first) {
                if ((rc = pcnn_persist_run(ctx, tmp, B, steps, nullptr, ctx->h_step_err + steps_done, fresh, last ? ctx->h_hs_done : nullptr,
                                           done_tag)))
                    return rc;
            } else {
                pcnn_persist_gate gate;
                gate.flags = ctx->d_hs_ready;
                gate.tag = ++ctx->hs_serial;
                if (gate.tag == 0) gate.tag = ++ctx->hs_serial;
                gate.chunks = ch;
                *ctx->h_hs_tag = gate.tag;   // the previous user of this word has been synchronised with (end of every launch)
                // The kernel goes first: it sets itself up while the host enqueues the copies, and waits on the flag of a
                // sample's chunk before it touches the sample.  Where kernel launches block the calling thread until the
                // kernel has finished (CUDA_LAUNCH_BLOCKING=1, profilers that replay kernels) the copies must be enqueued
                // before the launch instead, or the kernel would wait for chunks nobody can enqueue.
                const bool copies_first = ctx->hs_copies_first;
                if (!copies_first &&
                    (rc = pcnn_persist_run(ctx, tmp, B, steps, &gate, ctx->h_step_err + steps_done, fresh, last ? ctx->h_hs_done : nullptr,
                                           done_tag)))
                    return rc;
                PCNN_CUDA(cudaMemcpyAsync(ctx->d_hs_labels, host_labels + off, (size_t)sn, cudaMemcpyHostToDevice, ctx->copy_stream));
                long k = 0;
                for (long co = 0; co < sn; ++k) {
                    const long cs0 = (long)pcnn_chunk_size(ch, k);
                    const long cs = sn - co < cs0 ? sn - co : cs0;
                    PCNN_CUDA(cudaMemcpyAsync((char *)ctx->d_hs_images + (size_t)co * img_bytes, hi + (size_t)(off + co) * img_bytes,
                                              (size_t)cs * img_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
                    PCNN_CUDA(cudaMemcpyAsync(ctx->d_hs_ready + k, ctx->h_hs_tag, sizeof(unsigned), cudaMemcpyHostToDevice, ctx->copy_stream));
                    co += cs;
                }
                if (copies_first &&
                    (rc = pcnn_persist_run(ctx, tmp, B, steps, &gate, ctx->h_step_err + steps_done, fresh, last ? ctx->h_hs_done : nullptr,
                                           done_tag)))
                    return rc;
            }
            steps_done += steps;
            if (last) {
                if ((rc = wait_done_tag(ctx, done_tag))) return rc;
                err = ctx->h_hs_done[0];
            } else if (off + sn < n || !resident_after_first) {
                // the staging buffer is about to be refilled: wait for the kernel
                PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
                if ((rc = pcnn_persist_check(ctx))) return rc;
            }
        }
        ctx->step_err_count = steps_done;
    }
    if (mean_err_out) *mean_err_out = (float)(err / ((double)n * ctx->world));   // err is the all-reduced sum
    return PCNN_OK;
}

extern "C" int pcnn_learn_host(pcnn_ctx *ctx, const void *host_images, int pixel_type, const uint8_t *host_labels,
                               long n, int B, int epochs, float *mean_err_out) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_learn_host: ctx is NULL");
    PCNN_REQUIRE(host_images && host_labels && n > 0 && B > 0 && epochs > 0, PCNN_ERR_ARG, "pcnn_learn_host: bad arguments");
    PCNN_REQUIRE(pixel_type == PCNN_U8 || pixel_type == PCNN_F32, PCNN_ERR_ARG, "pcnn_learn_host: bad pixel type");
    pcnn_device_guard g(ctx->device);
    if (ctx->step_mode == PCNN_MODE_PERSISTENT)
        PCNN_REQUIRE(use_persistent(ctx), PCNN_ERR_STATE, "persistent mode requested but peers are not attached");
    if (use_persistent(ctx)) {
        // pinned + mapped + 16-byte aligned images: the kernel pulls them itself; pageable memory goes through the staged stream
        cudaPointerAttributes at{};
        const cudaError_t pe = cudaPointerGetAttributes(&at, host_images);
        if (pe != cudaSuccess) cudaGetLastError();
        if (pe == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer && ((uintptr_t)at.devicePointer & 15) == 0 &&
            !ctx->hs_no_pull)
            return learn_host_pull(ctx, at.devicePointer, pixel_type, host_labels, n, B, epochs, mean_err_out);
        return learn_host_streamed(ctx, host_images, pixel_type, host_labels, n, B, epochs, mean_err_out);
    }
    return learn_host_chunked(ctx, host_images, pixel_type, host_labels, n, B, epochs, mean_err_out);
}

// ------------------------------------------------------------------------------------------ C ABI: evaluation
extern "C" int pcnn_forward_batch(pcnn_ctx *ctx, const void *dev_images, int pixel_type, int B, float *f_out_dev,
                                  uint8_t *pred_dev) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_forward_batch: ctx is NULL");
    PCNN_REQUIRE(dev_images && B > 0, PCNN_ERR_ARG, "pcnn_forward_batch: NULL images or B <= 0");
    PCNN_REQUIRE(pixel_type == PCNN_U8 || pixel_type == PCNN_F32, PCNN_ERR_ARG, "pcnn_forward_batch: bad pixel type");
    PCNN_REQUIRE(((uintptr_t)dev_images & 15) == 0, PCNN_ERR_ARG, "pcnn_forward_batch: images must be 16-byte aligned");
    pcnn_device_guard g(ctx->device);
    FusedArgs a{};
    a.images = dev_images;
    a.params = ctx->d_params;
    a.f_out = f_out_dev;
    a.pred = pred_dev;
    a.n_total = B;
    a.B = B;
    a.world = 1;
    return launch_fused<false>(ctx, a, pixel_type, fused_grid(ctx, B));
}

extern "C" int pcnn_test(pcnn_ctx *ctx, long *wrong_out) {
    PCNN_REQUIRE(ctx && wrong_out, PCNN_ERR_ARG, "pcnn_test: NULL argument");
    const pcnn_split_binding &s = ctx->split[PCNN_TEST_SET];
    PCNN_REQUIRE(s.n > 0, PCNN_ERR_STATE, "pcnn_test: no test split bound");
    PCNN_REQUIRE(s.n <= 0x7fffffffL, PCNN_ERR_ARG, "pcnn_test: split too large");
    pcnn_device_guard g(ctx->device);
    PCNN_CUDA(cudaMemsetAsync(ctx->d_wrong, 0, sizeof(int), ctx->stream));
    FusedArgs a{};
    a.images = s.images;
    a.labels = s.labels;
    a.params = ctx->d_params;
    a.wrong = ctx->d_wrong;
    a.n_total = s.n;
    a.B = (int)s.n;
    a.world = 1;
    int rc = launch_fused<false>(ctx, a, s.pixel_type, fused_grid(ctx, (int)s.n));
    if (rc) return rc;
    int wrong = 0;
    PCNN_CUDA(cudaMemcpyAsync(ctx->h_scalar, ctx->d_wrong, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    wrong = *reinterpret_cast<int *>(ctx->h_scalar);
    *wrong_out = wrong;
    return PCNN_OK;
}

extern "C" int pcnn_step_errs(pcnn_ctx *ctx, float *host_out, long cap, long *count_out) {
    PCNN_REQUIRE(ctx && count_out, PCNN_ERR_ARG, "pcnn_step_errs: NULL argument");
    pcnn_device_guard g(ctx->device);
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    *count_out = ctx->step_err_count;
    if (host_out)
        for (long i = 0; i < ctx->step_err_count && i < cap; ++i) host_out[i] = ctx->h_step_err[i];
    return PCNN_OK;
}

// ------------------------------------------------------------------------------------------ measurement helpers
extern "C" int pcnn_time_fused_kernel(pcnn_ctx *ctx, int B, int iters, float *avg_ms_out) {
    PCNN_REQUIRE(ctx && avg_ms_out, PCNN_ERR_ARG, "pcnn_time_fused_kernel: NULL argument");
    const pcnn_split_binding &s = ctx->split[PCNN_TRAIN_SET];
    PCNN_REQUIRE(s.n >= B && B > 0 && iters > 0, PCNN_ERR_STATE, "pcnn_time_fused_kernel: bind a train split of at least B samples");
    pcnn_device_guard g(ctx->device);
    cudaEvent_t e0, e1;
    PCNN_CUDA(cudaEventCreate(&e0));
    PCNN_CUDA(cudaEventCreate(&e1));
    const long windows = s.n / B;
    int rc = PCNN_OK, grid = 0;
    long w = 0;
    for (int i = 0; i < iters / 10 + 3 && rc == PCNN_OK; ++i, w = (w + 1) % windows)
        rc = pcnn_launch_fused_grad(ctx, src_of(s, w * B, false), B, &grid);
    if (rc == PCNN_OK) {
        cudaEventRecord(e0, ctx->stream);
        for (int i = 0; i < iters && rc == PCNN_OK; ++i, w = (w + 1) % windows)
            rc = pcnn_launch_fused_grad(ctx, src_of(s, w * B, false), B, &grid);
        cudaEventRecord(e1, ctx->stream);
        cudaError_t e = cudaEventSynchronize(e1);
        float ms = 0.0f;
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, e0, e1);
        if (e != cudaSuccess) rc = pcnn_fail_cuda(e, "event timing", __FILE__, __LINE__);
        *avg_ms_out = ms / (float)iters;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return rc;
}

namespace {
// 8 independent FMA chains per thread, 4096 iterations: 65,536 FMAs per thread, no memory traffic
__global__ void __launch_bounds__(256) k_fma_peak(float *out, float a, float b) {
    float x0 = threadIdx.x, x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3, x4 = x0 + 4, x5 = x0 + 5, x6 = x0 + 6, x7 = x0 + 7;
#pragma unroll 1
    for (int i = 0; i < 256; ++i) {       // 256 FFMA per loop trip: loop overhead < 2 % of the issue slots
#pragma unroll
        for (int u = 0; u < 32; ++u) {
            x0 = fmaf(x0, a, b); x1 = fmaf(x1, a, b); x2 = fmaf(x2, a, b); x3 = fmaf(x3, a, b);
            x4 = fmaf(x4, a, b); x5 = fmaf(x5, a, b); x6 = fmaf(x6, a, b); x7 = fmaf(x7, a, b);
        }
    }
    if (x0 + x1 + x2 + x3 + x4 + x5 + x6 + x7 == 12345.678f) out[0] = x0;
}
}  // namespace

extern "C" int pcnn_measure_fp32_peak(pcnn_ctx *ctx, float *tflops_out) {
    PCNN_REQUIRE(ctx && tflops_out, PCNN_ERR_ARG, "pcnn_measure_fp32_peak: NULL argument");
    pcnn_device_guard g(ctx->device);
    cudaEvent_t e0, e1;
    PCNN_CUDA(cudaEventCreate(&e0));
    PCNN_CUDA(cudaEventCreate(&e1));
    const int grid = ctx->sm_count * 8, reps = 20;
    for (int i = 0; i < 3; ++i) k_fma_peak<<<grid, 256, 0, ctx->stream>>>(ctx->d_grads, 0.999f, 0.001f);
    cudaEventRecord(e0, ctx->stream);
    for (int i = 0; i < reps; ++i) k_fma_peak<<<grid, 256, 0, ctx->stream>>>(ctx->d_grads, 0.999f, 0.001f);
    cudaEventRecord(e1, ctx->stream);
    ctx->launches += reps + 3;
    PCNN_CUDA(cudaEventSynchronize(e1));
    float ms = 0.0f;
    PCNN_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    const double flops = 2.0 * 16.0 * 4096.0 * 256.0 * grid * reps;
    *tflops_out = (float)(flops / (ms * 1e-3) / 1e12);
    return PCNN_OK;
}
