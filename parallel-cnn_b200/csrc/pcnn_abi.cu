// parallel-cnn_b200/csrc/pcnn_abi.cu -- context, memory, parameters, data and checkpoint entry points of
// include/pcnn.h.  The kernels live in ops_kernels.cu / fused_kernels.cu / ext_kernels.cu.
#include "pcnn_internal.h"

#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

// --------------------------------------------------------------------------------------------- errors
static thread_local char g_err[512] = "no error";

void pcnn_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int pcnn_fail_cuda(cudaError_t e, const char *what, const char *file, int line) {
    pcnn_set_error("CUDA error %d (%s) at %s:%d in `%s`", (int)e, cudaGetErrorString(e), file, line, what);
    return PCNN_ERR_CUDA;
}

extern "C" int pcnn_version(void) { return PCNN_VERSION_NUMBER; }
extern "C" const char *pcnn_last_error_string(void) { return g_err; }

// --------------------------------------------------------------------------------------------- context
extern "C" int pcnn_create(pcnn_ctx **out, int device, void *stream) {
    PCNN_REQUIRE(out != nullptr, PCNN_ERR_ARG, "pcnn_create: out is NULL");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        pcnn_set_error("pcnn_create: no CUDA device available (%s); this engine has no CPU fallback",
                       e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
        cudaGetLastError();
        return PCNN_ERR_NOGPU;
    }
    if (device < 0) PCNN_CUDA(cudaGetDevice(&device));
    PCNN_REQUIRE(device < ndev, PCNN_ERR_ARG, "pcnn_create: device %d out of range (%d devices)", device, ndev);
    cudaDeviceProp prop;
    PCNN_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        pcnn_set_error("pcnn_create: device %d is sm_%d%d; libpcnn.so carries sm_90a code only", device,
                       prop.major, prop.minor);
        return PCNN_ERR_NOGPU;
    }
    PCNN_CUDA(cudaSetDevice(device));
    pcnn_ctx *c = new pcnn_ctx();
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    c->cc_major = prop.major;
    c->cc_minor = prop.minor;
    c->hbm_bytes = prop.totalGlobalMem;
    if (stream) {
        c->stream = (cudaStream_t)stream;
    } else {
        PCNN_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
        c->own_stream = true;
    }
    PCNN_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
        PCNN_CUDA(cudaEventCreateWithFlags(&c->ev_copy[i], cudaEventDisableTiming));
        PCNN_CUDA(cudaEventCreateWithFlags(&c->ev_done[i], cudaEventDisableTiming));
    }
    PCNN_CUDA(cudaMalloc(&c->d_params, NPACK * sizeof(float)));
    PCNN_CUDA(cudaMalloc(&c->d_grads, NPACK * sizeof(float)));
    PCNN_CUDA(cudaMalloc(&c->d_slots, (size_t)MAX_SLOTS * NPACK * sizeof(float)));
    PCNN_CUDA(cudaMalloc(&c->d_err_total, sizeof(double)));
    PCNN_CUDA(cudaMalloc(&c->d_cursor, sizeof(long long)));
    PCNN_CUDA(cudaMalloc(&c->d_wrong, sizeof(int)));
    PCNN_CUDA(cudaMalloc(&c->d_step_err, STEP_ERR_CAP * sizeof(float)));
    PCNN_CUDA(cudaMemset(c->d_step_err, 0, STEP_ERR_CAP * sizeof(float)));
    PCNN_CUDA(cudaMalloc(&c->d_step_idx, sizeof(int)));
    PCNN_CUDA(cudaMemset(c->d_step_idx, 0, sizeof(int)));
    PCNN_CUDA(cudaMalloc(&c->d_abort, sizeof(int)));
    PCNN_CUDA(cudaMemset(c->d_abort, 0, sizeof(int)));
    PCNN_CUDA(cudaMemset(c->d_params, 0, NPACK * sizeof(float)));
    PCNN_CUDA(cudaMemset(c->d_grads, 0, NPACK * sizeof(float)));
    PCNN_CUDA(cudaMemset(c->d_err_total, 0, sizeof(double)));
    PCNN_CUDA(cudaMemset(c->d_cursor, 0, sizeof(long long)));
    PCNN_CUDA(cudaMemset(c->d_wrong, 0, sizeof(int)));
    PCNN_CUDA(cudaMallocHost(&c->h_scalar, 64));
    {
        int rc = pcnn_fused_configure();
        if (rc) return rc;
        if ((rc = pcnn_persist_configure(c))) return rc;
    }
    {   // a CUDA runtime setting, not a knob of this library: blocking launches change the order pcnn_learn_host must enqueue in
        const char *lb = getenv("CUDA_LAUNCH_BLOCKING");
        c->hs_copies_first = lb && lb[0] == '1';
    }
    // default parameters = the reference's static-constructor state
    float init[NPARAM];
    pcnn_init_params_reference(init);
    PCNN_CUDA(cudaMemcpy(c->d_params, init, sizeof(init), cudaMemcpyHostToDevice));
    *out = c;
    return PCNN_OK;
}

static void release_split(pcnn_split_binding &s) {
    if (s.owned_images) cudaFree(s.owned_images);
    if (s.owned_labels) cudaFree(s.owned_labels);
    s = pcnn_split_binding();
}

extern "C" int pcnn_destroy(pcnn_ctx *ctx) {
    if (!ctx) return PCNN_OK;
    pcnn_device_guard g(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    pcnn_comm_destroy(ctx);
    pcnn_p2p_detach(ctx);
    if (ctx->p2p_base) cudaFree(ctx->p2p_base);
    if (ctx->scratch) cudaFree(ctx->scratch);
    if (ctx->scratch2) cudaFree(ctx->scratch2);
    if (ctx->d_trace) cudaFree(ctx->d_trace);
    if (ctx->d_hs_images) cudaFree(ctx->d_hs_images);
    if (ctx->d_hs_labels) cudaFree(ctx->d_hs_labels);
    if (ctx->d_hs_ready) cudaFree(ctx->d_hs_ready);
    if (ctx->h_hs_tag) cudaFreeHost(ctx->h_hs_tag);
    if (ctx->h_hs_done) cudaFreeHost(ctx->h_hs_done);
    if (ctx->d_slots_ll) cudaFree(ctx->d_slots_ll);
    if (ctx->d_params_ll) cudaFree(ctx->d_params_ll);
    if (ctx->d_abort) cudaFree(ctx->d_abort);
    for (auto &kv : ctx->graphs) cudaGraphExecDestroy(kv.second);
    ctx->graphs.clear();
    release_split(ctx->split[0]);
    release_split(ctx->split[1]);
    for (int i = 0; i < 2; ++i) {
        if (ctx->h_stage[i]) cudaFreeHost(ctx->h_stage[i]);
        if (ctx->d_stage[i]) cudaFree(ctx->d_stage[i]);
        if (ctx->h_stage_lab[i]) cudaFreeHost(ctx->h_stage_lab[i]);
        if (ctx->d_stage_lab[i]) cudaFree(ctx->d_stage_lab[i]);
        if (ctx->ev_copy[i]) cudaEventDestroy(ctx->ev_copy[i]);
        if (ctx->ev_done[i]) cudaEventDestroy(ctx->ev_done[i]);
    }
    if (ctx->h_scalar) cudaFreeHost(ctx->h_scalar);
    cudaFree(ctx->d_params);
    cudaFree(ctx->d_grads);
    cudaFree(ctx->d_slots);
    cudaFree(ctx->d_err_total);
    cudaFree(ctx->d_cursor);
    cudaFree(ctx->d_wrong);
    if (ctx->d_step_err) cudaFree(ctx->d_step_err);
    if (ctx->d_step_idx) cudaFree(ctx->d_step_idx);
    if (ctx->h_step_err) cudaFreeHost(ctx->h_step_err);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
    return PCNN_OK;
}

int pcnn_scratch(pcnn_ctx *ctx, size_t bytes, void **out) {
    if (bytes > ctx->scratch_bytes) {
        PCNN_CUDA(cudaStreamSynchronize(ctx->stream));       // earlier work may still be using the old block
        if (ctx->scratch) PCNN_CUDA(cudaFree(ctx->scratch));
        ctx->scratch = nullptr;
        ctx->scratch_bytes = 0;
        const size_t want = (bytes + ((size_t)1 << 20) - 1) & ~(((size_t)1 << 20) - 1);
        PCNN_CUDA(cudaMalloc(&ctx->scratch, want));
        ctx->scratch_bytes = want;
    }
    *out = ctx->scratch;
    return PCNN_OK;
}

extern "C" int pcnn_sync(pcnn_ctx *ctx) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_sync: ctx is NULL");
    pcnn_device_guard g(ctx->device);
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    return pcnn_persist_check(ctx);
}

extern "C" int pcnn_device_info(pcnn_ctx *ctx, int *sm_count, int *cc_major, int *cc_minor, size_t *hbm_bytes) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_device_info: ctx is NULL");
    if (sm_count) *sm_count = ctx->sm_count;
    if (cc_major) *cc_major = ctx->cc_major;
    if (cc_minor) *cc_minor = ctx->cc_minor;
    if (hbm_bytes) *hbm_bytes = ctx->hbm_bytes;
    return PCNN_OK;
}

extern "C" int pcnn_launch_count(pcnn_ctx *ctx, long *count_out) {
    PCNN_REQUIRE(ctx && count_out, PCNN_ERR_ARG, "pcnn_launch_count: NULL argument");
    *count_out = ctx->launches;
    return PCNN_OK;
}

// --------------------------------------------------------------------------------------------- buffers
extern "C" int pcnn_malloc(pcnn_ctx *ctx, void **dev, size_t bytes) {
    PCNN_REQUIRE(ctx && dev, PCNN_ERR_ARG, "pcnn_malloc: NULL argument");
    pcnn_device_guard g(ctx->device);
    *dev = nullptr;
    if (bytes == 0) bytes = 4;   // Layer(0, 0, O) allocates zero-length arrays (layer.h:42-43)
    PCNN_CUDA(cudaMalloc(dev, bytes));
    PCNN_CUDA(cudaMemsetAsync(*dev, 0, bytes, ctx->stream));
    return PCNN_OK;
}
extern "C" int pcnn_free(pcnn_ctx *ctx, void *dev) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_free: ctx is NULL");
    pcnn_device_guard g(ctx->device);
    if (dev) {
        PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
        PCNN_CUDA(cudaFree(dev));
    }
    return PCNN_OK;
}
extern "C" int pcnn_memset0(pcnn_ctx *ctx, void *dev, size_t bytes) {
    PCNN_REQUIRE(ctx && (dev || bytes == 0), PCNN_ERR_ARG, "pcnn_memset0: NULL argument");
    pcnn_device_guard g(ctx->device);
    if (bytes) PCNN_CUDA(cudaMemsetAsync(dev, 0, bytes, ctx->stream));
    return PCNN_OK;
}
extern "C" int pcnn_h2d(pcnn_ctx *ctx, void *dev, const void *host, size_t bytes) {
    PCNN_REQUIRE(ctx && (bytes == 0 || (dev && host)), PCNN_ERR_ARG, "pcnn_h2d: NULL argument");
    pcnn_device_guard g(ctx->device);
    if (bytes) {
        PCNN_CUDA(cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
        PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    return PCNN_OK;
}
extern "C" int pcnn_d2h(pcnn_ctx *ctx, void *host, const void *dev, size_t bytes) {
    PCNN_REQUIRE(ctx && (bytes == 0 || (dev && host)), PCNN_ERR_ARG, "pcnn_d2h: NULL argument");
    pcnn_device_guard g(ctx->device);
    if (bytes) {
        PCNN_CUDA(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    return PCNN_OK;
}
extern "C" int pcnn_d2d(pcnn_ctx *ctx, void *dst, const void *src, size_t bytes) {
    PCNN_REQUIRE(ctx && (bytes == 0 || (dst && src)), PCNN_ERR_ARG, "pcnn_d2d: NULL argument");
    pcnn_device_guard g(ctx->device);
    if (bytes) PCNN_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    return PCNN_OK;
}

// --------------------------------------------------------------------------------------------- parameters
// glibc's default rand() is random_r TYPE_3: a 31-word additive feedback generator r[i] = r[i-3] + r[i-31]
// seeded through the Lehmer step 16807 * x mod (2^31 - 1), first 310 outputs discarded, result >> 1.
// Re-implemented privately so the library never touches the process-wide rand() state; tests/ check it
// against the real rand() and against the reference's constructed weights (golden params_init).
namespace {
struct glibc_rand {
    uint32_t r[34 + 310 + 3000];
    int next;
    explicit glibc_rand(uint32_t seed, int n_outputs) {
        int32_t word = (int32_t)(seed ? seed : 1);
        r[0] = (uint32_t)word;
        for (int i = 1; i < 31; ++i) {
            long hi = word / 127773, lo = word % 127773;
            word = (int32_t)(16807 * lo - 2836 * hi);
            if (word < 0) word += 2147483647;
            r[i] = (uint32_t)word;
        }
        for (int i = 31; i < 34; ++i) r[i] = r[i - 31];
        for (int i = 34; i < 344 + n_outputs; ++i) r[i] = r[i - 31] + r[i - 3];
        next = 344;
    }
    int operator()() { return (int)(r[next++] >> 1); }
};
}  // namespace

extern "C" int pcnn_init_params_reference(float *p) {
    PCNN_REQUIRE(p, PCNN_ERR_ARG, "pcnn_init_params_reference: NULL output");
    glibc_rand rnd(1, NPARAM);
    const float rand_max = (float)2147483647;   // RAND_MAX converted to float, as in `float / int` (layer.h:49)
    auto draw = [&](float *w, float *b, int M, int N) {
        for (int n = 0; n < N; ++n) {
            b[n] = 0.5f - (float)rnd() / rand_max;
            for (int k = 0; k < M; ++k) w[n * M + k] = 0.5f - (float)rnd() / rand_max;
        }
    };
    draw(p + OFF_C1W, p + OFF_C1B, 25, 6);     // l_c1(5*5, 6, 24*24*6)   Main.cpp:18
    draw(p + OFF_S1W, p + OFF_S1B, 16, 1);     // l_s1(4*4, 1, 6*6*6)     Main.cpp:19
    draw(p + OFF_FW, p + OFF_FB, 216, 10);     // l_f(6*6*6, 10, 10)      Main.cpp:20
    return PCNN_OK;
}

extern "C" int pcnn_set_params(pcnn_ctx *ctx, const float *host_params) {
    PCNN_REQUIRE(ctx && host_params, PCNN_ERR_ARG, "pcnn_set_params: NULL argument");
    pcnn_device_guard g(ctx->device);
    PCNN_CUDA(cudaMemcpyAsync(ctx->d_params, host_params, NPARAM * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    return PCNN_OK;
}
extern "C" int pcnn_get_params(pcnn_ctx *ctx, float *host_params) {
    PCNN_REQUIRE(ctx && host_params, PCNN_ERR_ARG, "pcnn_get_params: NULL argument");
    return pcnn_d2h(ctx, host_params, ctx->d_params, NPARAM * sizeof(float));
}
extern "C" int pcnn_get_grads(pcnn_ctx *ctx, float *host_grads) {
    PCNN_REQUIRE(ctx && host_grads, PCNN_ERR_ARG, "pcnn_get_grads: NULL argument");
    return pcnn_d2h(ctx, host_grads, ctx->d_grads, NPARAM * sizeof(float));
}
extern "C" int pcnn_params_dev(pcnn_ctx *ctx, float **dev_params) {
    PCNN_REQUIRE(ctx && dev_params, PCNN_ERR_ARG, "pcnn_params_dev: NULL argument");
    *dev_params = ctx->d_params;
    return PCNN_OK;
}
extern "C" int pcnn_set_learning_rate(pcnn_ctx *ctx, float dt) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_set_learning_rate: ctx is NULL");
    ctx->lr = dt;
    // graphs bake the step size into kernel arguments
    pcnn_device_guard g(ctx->device);
    for (auto &kv : ctx->graphs) cudaGraphExecDestroy(kv.second);
    ctx->graphs.clear();
    return PCNN_OK;
}
extern "C" int pcnn_err_sum(pcnn_ctx *ctx, double *sum_out, int reset) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_err_sum: ctx is NULL");
    pcnn_device_guard g(ctx->device);
    if (sum_out) {
        PCNN_CUDA(cudaMemcpyAsync(sum_out, ctx->d_err_total, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
        int rc = pcnn_persist_check(ctx);
        if (rc) return rc;
    }
    if (reset) PCNN_CUDA(cudaMemsetAsync(ctx->d_err_total, 0, sizeof(double), ctx->stream));
    return PCNN_OK;
}

// checkpoint: "PCNN" magic, version, count, reserved, then 2,343 little-endian fp32 in packed order
struct ckpt_header { char magic[4]; uint32_t version, count, reserved; };

extern "C" int pcnn_save_params(pcnn_ctx *ctx, const char *path) {
    PCNN_REQUIRE(ctx && path, PCNN_ERR_ARG, "pcnn_save_params: NULL argument");
    float p[NPARAM];
    int rc = pcnn_get_params(ctx, p);
    if (rc) return rc;
    FILE *f = fopen(path, "wb");
    PCNN_REQUIRE(f, PCNN_ERR_IO, "pcnn_save_params: cannot open %s for writing", path);
    ckpt_header h = {{'P', 'C', 'N', 'N'}, 1u, (uint32_t)NPARAM, 0u};
    bool ok = fwrite(&h, sizeof(h), 1, f) == 1 && fwrite(p, sizeof(float), NPARAM, f) == (size_t)NPARAM;
    ok = (fclose(f) == 0) && ok;
    PCNN_REQUIRE(ok, PCNN_ERR_IO, "pcnn_save_params: short write to %s", path);
    return PCNN_OK;
}
extern "C" int pcnn_load_params(pcnn_ctx *ctx, const char *path) {
    PCNN_REQUIRE(ctx && path, PCNN_ERR_ARG, "pcnn_load_params: NULL argument");
    FILE *f = fopen(path, "rb");
    PCNN_REQUIRE(f, PCNN_ERR_IO, "pcnn_load_params: cannot open %s", path);
    ckpt_header h;
    float p[NPARAM];
    bool ok = fread(&h, sizeof(h), 1, f) == 1 && memcmp(h.magic, "PCNN", 4) == 0 && h.version == 1 &&
              h.count == (uint32_t)NPARAM && fread(p, sizeof(float), NPARAM, f) == (size_t)NPARAM;
    fclose(f);
    PCNN_REQUIRE(ok, PCNN_ERR_IO, "pcnn_load_params: %s is not a valid parameter file", path);
    return pcnn_set_params(ctx, p);
}

// --------------------------------------------------------------------------------------------- data
static unsigned be32(const unsigned char *b) {
    return ((unsigned)b[0] << 24) | ((unsigned)b[1] << 16) | ((unsigned)b[2] << 8) | (unsigned)b[3];
}

// IDX reader with mnist_load's contract (mnist.h:79-160): same checks in the same order, same return codes;
// short reads (which the reference ignores) are reported as the corresponding "not a valid file" code.
extern "C" int pcnn_mnist_load_u8(const char *image_file, const char *label_file, uint8_t **images,
                                  uint8_t **labels, unsigned *count) {
    PCNN_REQUIRE(image_file && label_file && images && labels && count, PCNN_ERR_ARG,
                 "pcnn_mnist_load_u8: NULL argument");
    *images = nullptr;
    *labels = nullptr;
    *count = 0;
    FILE *ifp = fopen(image_file, "rb");
    FILE *lfp = fopen(label_file, "rb");
    int rc = 0;
    unsigned char ih[16], lh[8];
    unsigned n = 0;
    uint8_t *img = nullptr, *lab = nullptr;
    if (!ifp || !lfp) { rc = -1; goto done; }                                   // no such files
    if (fread(ih, 1, 16, ifp) != 16 || be32(ih) != 2051) { rc = -2; goto done; }  // not a valid image file
    if (fread(lh, 1, 8, lfp) != 8 || be32(lh) != 2049) { rc = -3; goto done; }     // not a valid label file
    n = be32(ih + 4);
    if (n != be32(lh + 4)) { rc = -4; goto done; }                              // element counts mismatch
    if (be32(ih + 8) != 28 || be32(ih + 12) != 28) { rc = -2; goto done; }
    img = (uint8_t *)malloc((size_t)n * PCNN_IMG + 16);
    lab = (uint8_t *)malloc((size_t)n + 16);
    if (!img || !lab) { rc = PCNN_ERR_IO; goto done; }
    if (fread(img, PCNN_IMG, n, ifp) != n) { rc = -2; goto done; }
    if (fread(lab, 1, n, lfp) != n) { rc = -3; goto done; }
    *images = img;
    *labels = lab;
    *count = n;
    img = lab = nullptr;
done:
    if (ifp) fclose(ifp);
    if (lfp) fclose(lfp);
    free(img);
    free(lab);
    if (rc) pcnn_set_error("pcnn_mnist_load_u8(%s, %s): code %d", image_file, label_file, rc);
    return rc;
}
extern "C" void pcnn_mnist_free(void *p) { free(p); }

static size_t pixel_bytes(int pixel_type) { return pixel_type == PCNN_F32 ? sizeof(float) : 1; }

extern "C" int pcnn_dataset_bind(pcnn_ctx *ctx, int split, const void *dev_images, int pixel_type,
                                 const uint8_t *dev_labels, long n) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_dataset_bind: ctx is NULL");
    PCNN_REQUIRE(split == PCNN_TRAIN_SET || split == PCNN_TEST_SET, PCNN_ERR_ARG, "pcnn_dataset_bind: bad split %d", split);
    PCNN_REQUIRE(pixel_type == PCNN_U8 || pixel_type == PCNN_F32, PCNN_ERR_ARG, "pcnn_dataset_bind: bad pixel type %d", pixel_type);
    PCNN_REQUIRE(n >= 0 && (n == 0 || (dev_images && dev_labels)), PCNN_ERR_ARG, "pcnn_dataset_bind: NULL buffers with n=%ld", n);
    PCNN_REQUIRE(((uintptr_t)dev_images & 15) == 0, PCNN_ERR_ARG, "pcnn_dataset_bind: images must be 16-byte aligned");
    pcnn_device_guard g(ctx->device);
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    pcnn_drop_graphs(ctx);                 // graphs captured over the old buffers must not be replayed
    release_split(ctx->split[split]);
    ctx->split[split].images = dev_images;
    ctx->split[split].labels = dev_labels;
    ctx->split[split].pixel_type = pixel_type;
    ctx->split[split].n = n;
    return PCNN_OK;
}

extern "C" int pcnn_dataset_upload(pcnn_ctx *ctx, int split, const void *host_images, int pixel_type,
                                   const uint8_t *host_labels, long n) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_dataset_upload: ctx is NULL");
    PCNN_REQUIRE(split == PCNN_TRAIN_SET || split == PCNN_TEST_SET, PCNN_ERR_ARG, "pcnn_dataset_upload: bad split %d", split);
    PCNN_REQUIRE(pixel_type == PCNN_U8 || pixel_type == PCNN_F32, PCNN_ERR_ARG, "pcnn_dataset_upload: bad pixel type %d", pixel_type);
    PCNN_REQUIRE(n > 0 && host_images && host_labels, PCNN_ERR_ARG, "pcnn_dataset_upload: empty or NULL dataset");
    pcnn_device_guard g(ctx->device);
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));
    void *di = nullptr, *dl = nullptr;
    size_t ib = (size_t)n * PCNN_IMG * pixel_bytes(pixel_type);
    PCNN_CUDA(cudaMalloc(&di, ib + 16));
    PCNN_CUDA(cudaMalloc(&dl, (size_t)n + 16));
    PCNN_CUDA(cudaMemcpy(di, host_images, ib, cudaMemcpyHostToDevice));
    PCNN_CUDA(cudaMemcpy(dl, host_labels, (size_t)n, cudaMemcpyHostToDevice));
    pcnn_drop_graphs(ctx);                 // graphs captured over the old buffers must not be replayed
    release_split(ctx->split[split]);
    ctx->split[split].images = di;
    ctx->split[split].labels = (const uint8_t *)dl;
    ctx->split[split].owned_images = di;
    ctx->split[split].owned_labels = dl;
    ctx->split[split].pixel_type = pixel_type;
    ctx->split[split].n = n;
    return PCNN_OK;
}
