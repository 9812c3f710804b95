// parallel-cnn_b200/csrc/optim.cu -- momentum SGD and AdamW for device-trained layers (pcnn_optim_*): one launch updates every
// parameter tensor of a network and writes the bf16 operand of each wide or linear plan from the new fp32 master in the same pass.
// The contract, with the order of every operation, is in include/pcnn.h.
//
// Table.  pcnn_optim_create validates the tensors once and uploads one OptEntry per tensor (param, grad, state, plan operand and
// bias copy, weight decay, path) and a chunk table: tensor t owns the chunks [chunk0, chunk0 + ceil(n / OPT_CHUNK)), and entry c of
// the table is the tensor of chunk c.  CTA b takes chunks b, b + grid, ...; the update is element-wise, so the partition changes no
// bit.  Row-Toeplitz plans cannot be written element by element (one filter element feeds V * Qt operand entries): their filters are
// gathered by pcnn_conv_plan_set_params right after the update kernel.
#include "pcnn_internal.h"

#include <cuda_bf16.h>

#include <algorithm>
#include <cmath>
#include <vector>

namespace {

constexpr int OPT_THREADS = 256;
constexpr int OPT_CHUNK = 4096;           // elements per chunk: 4 float4 per thread on the vector path
constexpr int OPT_CTAS_PER_SM = 4;

struct OptEntry {
    float *p;
    const float *g;
    float *s0, *s1;                       // momentum buffer, or m and v; null where the kind keeps none
    __nv_bfloat16 *dst;                   // plan operand: element i at dst[(i / cols) * pitch + i % cols]; null without one
    float *mirror;                        // the plan's fp32 bias copy; null without one
    long long n, chunk0;
    float wd;
    int cols, pitch, vec;
};

// per-step scalars, formed on the host (pcnn_optim_step)
struct OptStep {
    float neg_lr, lr;
    float mu, omega;                      // SGD: momentum and fp32(1 - dampening)
    int momentum, first;                  // SGD: mu != 0; t == 1
    float a1, beta2, a2, eps, c2, neg_s;  // AdamW
};

__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }

// RN(a / b) for fp32 a, b without the out-of-line slow path of __fdiv_rn (its call convention puts the AdamW kernel on the stack).
// In double every fp32 quotient is far from overflow and underflow, and a double reciprocal from rcp.approx (about 23 bits; every
// nonzero fp32 is a normal double, so ftz never applies) refined by two Newton steps and one remainder step gives a quotient
// within one double ulp.  An fp32 quotient that is not a midpoint of fp32 (normal or subnormal) values lies at least 2^-49 of its
// size (normal) or 2^-173 (subnormal) away from one, more than that error, so rounding it to fp32 gives RN(a / b).  Zeros,
// infinities and NaN take a * (1 / b) in double, which gives IEEE's answer for each (and keeps the sign of a zero).
__device__ __forceinline__ float div_rn(float a, float b) {
    const double A = a, B = b;
    double y;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(B));
    if (a == 0.0f || !isfinite(a) || !isfinite(b) || b == 0.0f) return __double2float_rn(A * y);
    double e = fma(-B, y, 1.0);
    y = fma(y, e, y);
    e = fma(-B, y, 1.0);
    y = fma(y, e, y);
    const double q = A * y;
    return __double2float_rn(fma(fma(-B, q, A), y, q));
}

// one element of the rules in pcnn.h; lam = fp32(1 - lr * wd) (AdamW)
template <int KIND, bool NEST>
__device__ __forceinline__ void update(float &p, float g, float &s0, float &s1, float wd, float lam, const OptStep &s) {
    if (KIND == PCNN_OPTIM_SGD) {
        const float gp = wd != 0.0f ? add(g, mul(wd, p)) : g;
        float d = gp;
        if (s.momentum) {
            s0 = s.first ? gp : add(mul(s.mu, s0), mul(s.omega, gp));
            d = NEST ? add(gp, mul(s.mu, s0)) : s0;
        }
        p = add(p, mul(s.neg_lr, d));
    } else {
        if (wd != 0.0f) p = mul(p, lam);
        s0 = add(s0, mul(s.a1, __fsub_rn(g, s0)));
        s1 = add(mul(s.beta2, s1), mul(mul(s.a2, g), g));
        const float den = add(div_rn(__fsqrt_rn(s1), s.c2), s.eps);
        p = add(p, mul(s.neg_s, div_rn(s0, den)));
    }
}

template <int KIND>
__device__ __forceinline__ bool has_s0(const OptStep &s) { return KIND == PCNN_OPTIM_ADAMW || s.momentum; }

template <int KIND, bool NEST>
__global__ void __launch_bounds__(OPT_THREADS) k_optim(const OptEntry *__restrict__ tab, const int *__restrict__ chunk_tensor, int nchunks,
                                                       const OptStep s) {
    for (int c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const OptEntry e = tab[chunk_tensor[c]];
        const long long i0 = (c - e.chunk0) * (long long)OPT_CHUNK;
        const long long i1 = i0 + OPT_CHUNK < e.n ? i0 + OPT_CHUNK : e.n;
        const float lam = KIND == PCNN_OPTIM_ADAMW ? (float)(1.0 - (double)s.lr * (double)e.wd) : 1.0f;
        const bool st0 = has_s0<KIND>(s), st1 = KIND == PCNN_OPTIM_ADAMW;
        if (e.vec) {
            // i0 and n are multiples of 4, so every float4 is whole; with cols % 4 == 0 its 4 operand elements share a row
            for (long long i = i0 + 4 * threadIdx.x; i < i1; i += 4 * OPT_THREADS) {
                float4 p = *reinterpret_cast<const float4 *>(e.p + i);
                const float4 g = *reinterpret_cast<const float4 *>(e.g + i);
                float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
                if (st0) a = *reinterpret_cast<const float4 *>(e.s0 + i);
                if (st1) b = *reinterpret_cast<const float4 *>(e.s1 + i);
                update<KIND, NEST>(p.x, g.x, a.x, b.x, e.wd, lam, s);
                update<KIND, NEST>(p.y, g.y, a.y, b.y, e.wd, lam, s);
                update<KIND, NEST>(p.z, g.z, a.z, b.z, e.wd, lam, s);
                update<KIND, NEST>(p.w, g.w, a.w, b.w, e.wd, lam, s);
                *reinterpret_cast<float4 *>(e.p + i) = p;
                if (st0) *reinterpret_cast<float4 *>(e.s0 + i) = a;
                if (st1) *reinterpret_cast<float4 *>(e.s1 + i) = b;
                if (e.dst) {
                    const __nv_bfloat162 lo = __floats2bfloat162_rn(p.x, p.y), hi = __floats2bfloat162_rn(p.z, p.w);
                    uint2 v;
                    v.x = *reinterpret_cast<const unsigned *>(&lo);
                    v.y = *reinterpret_cast<const unsigned *>(&hi);
                    *reinterpret_cast<uint2 *>(e.dst + (i / e.cols) * e.pitch + i % e.cols) = v;
                }
                if (e.mirror) *reinterpret_cast<float4 *>(e.mirror + i) = p;
            }
        } else {
            for (long long i = i0 + threadIdx.x; i < i1; i += OPT_THREADS) {
                float p = e.p[i], a = 0.0f, b = 0.0f;
                if (st0) a = e.s0[i];
                if (st1) b = e.s1[i];
                update<KIND, NEST>(p, e.g[i], a, b, e.wd, lam, s);
                e.p[i] = p;
                if (st0) e.s0[i] = a;
                if (st1) e.s1[i] = b;
                if (e.dst) e.dst[(i / e.cols) * e.pitch + i % e.cols] = __float2bfloat16_rn(p);
                if (e.mirror) e.mirror[i] = p;
            }
        }
    }
}

bool aligned(const void *p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

}  // namespace

struct pcnn_optim {
    pcnn_optim_config cfg;
    int count = 0, nchunks = 0, grid = 0, nvec = 0;
    long long elements = 0, steps = 0;
    std::vector<OptEntry> host;           // the uploaded table (device pointers), for pcnn_optim_state
    std::vector<pcnn_conv_plan *> toeplitz;   // row-Toeplitz plans with their filters in the table, refreshed after each update
    std::vector<float *> toeplitz_filt;
    OptEntry *d_tab = nullptr;
    int *d_chunks = nullptr;
    float *d_state = nullptr;
};

static void free_optim(pcnn_optim *o) {
    if (!o) return;
    if (o->d_tab) cudaFree(o->d_tab);
    if (o->d_chunks) cudaFree(o->d_chunks);
    if (o->d_state) cudaFree(o->d_state);
    delete o;
}

static int check_config(const pcnn_optim_config *c) {
    const char *fn = "pcnn_optim_create";
    PCNN_REQUIRE(c->kind == PCNN_OPTIM_SGD || c->kind == PCNN_OPTIM_ADAMW, PCNN_ERR_ARG,
                 "%s: kind %d is not PCNN_OPTIM_SGD (0) or PCNN_OPTIM_ADAMW (1)", fn, c->kind);
    if (c->kind == PCNN_OPTIM_SGD) {
        PCNN_REQUIRE(!std::isnan(c->momentum) && !std::isnan(c->dampening), PCNN_ERR_ARG, "%s: momentum or dampening is NaN", fn);
        PCNN_REQUIRE(c->momentum >= 0.0f, PCNN_ERR_ARG, "%s: momentum %g < 0", fn, (double)c->momentum);
        PCNN_REQUIRE(!c->nesterov || (c->momentum > 0.0f && c->dampening == 0.0f), PCNN_ERR_ARG,
                     "%s: nesterov needs momentum > 0 and dampening 0 (momentum %g, dampening %g)", fn, (double)c->momentum,
                     (double)c->dampening);
    } else {
        PCNN_REQUIRE(!std::isnan(c->beta1) && !std::isnan(c->beta2) && !std::isnan(c->eps), PCNN_ERR_ARG, "%s: beta1, beta2 or eps is NaN",
                     fn);
        PCNN_REQUIRE(c->beta1 >= 0.0f && c->beta1 < 1.0f && c->beta2 >= 0.0f && c->beta2 < 1.0f, PCNN_ERR_ARG,
                     "%s: betas (%g, %g) outside [0, 1)", fn, (double)c->beta1, (double)c->beta2);
        PCNN_REQUIRE(c->eps >= 0.0f, PCNN_ERR_ARG, "%s: eps %g < 0", fn, (double)c->eps);
    }
    return PCNN_OK;
}

extern "C" int pcnn_optim_create(pcnn_ctx *ctx, const pcnn_optim_config *cfg, const pcnn_optim_tensor *t, int count, pcnn_optim **out) {
    const char *fn = "pcnn_optim_create";
    PCNN_REQUIRE(ctx && cfg && t && out, PCNN_ERR_ARG, "%s: NULL argument", fn);
    PCNN_REQUIRE(count >= 1, PCNN_ERR_ARG, "%s: count %d < 1", fn, count);
    int rc = check_config(cfg);
    if (rc) return rc;
    const int kind = cfg->kind;
    const bool st0 = kind == PCNN_OPTIM_ADAMW || cfg->momentum != 0.0f, st1 = kind == PCNN_OPTIM_ADAMW;
    struct Range { uintptr_t lo, hi; int tensor; const char *what; };
    std::vector<Range> ranges;
    std::vector<OptEntry> tab(count);
    long long chunks = 0, elements = 0, state_floats = 0;
    for (int i = 0; i < count; ++i) {
        const pcnn_optim_tensor &x = t[i];
        PCNN_REQUIRE(x.param && x.grad, PCNN_ERR_ARG, "%s: tensor %d: NULL param or grad", fn, i);
        PCNN_REQUIRE(x.n > 0, PCNN_ERR_ARG, "%s: tensor %d: n = %ld <= 0", fn, i, x.n);
        PCNN_REQUIRE(!std::isnan(x.weight_decay), PCNN_ERR_ARG, "%s: tensor %d: weight_decay is NaN", fn, i);
        PCNN_REQUIRE(x.weight_decay >= 0.0f, PCNN_ERR_ARG, "%s: tensor %d: weight_decay %g < 0", fn, i, (double)x.weight_decay);
        PCNN_REQUIRE(x.plan_part >= 0 && x.plan_part <= 2, PCNN_ERR_ARG, "%s: tensor %d: plan_part %d is not 0 (none), 1 (filters) or 2 (bias)",
                     fn, i, x.plan_part);
        PCNN_REQUIRE((x.plan_part == 0) == (x.plan == nullptr), PCNN_ERR_ARG,
                     "%s: tensor %d: plan_part %d %s a plan", fn, i, x.plan_part, x.plan ? "with" : "without");
        OptEntry &e = tab[i];
        e = OptEntry{x.param, x.grad, nullptr, nullptr, nullptr, nullptr, x.n, chunks, x.weight_decay, 1, 1, 0};
        const size_t bytes = (size_t)x.n * sizeof(float);
        ranges.push_back({(uintptr_t)x.param, (uintptr_t)x.param + bytes, i, "param"});
        ranges.push_back({(uintptr_t)x.grad, (uintptr_t)x.grad + bytes, i, "grad"});
        bool vec_ok = x.n % 4 == 0 && aligned(x.param, 16) && aligned(x.grad, 16);
        if (x.plan) {
            for (int j = 0; j < i; ++j)
                PCNN_REQUIRE(!(t[j].plan == x.plan && t[j].plan_part == x.plan_part), PCNN_ERR_ARG,
                             "%s: tensors %d and %d: the same plan part (%d) listed twice", fn, j, i, x.plan_part);
            const pcnn_conv_plan &pl = *x.plan;
            if (x.plan_part == 1) {
                PCNN_REQUIRE(x.n == pl.n, PCNN_ERR_ARG, "%s: tensor %d: n = %ld, but the plan's filters / weights have %lld elements", fn, i,
                             x.n, pl.n);
                if (pl.w) {
                    e.dst = static_cast<__nv_bfloat16 *>(pl.w);
                    e.cols = pl.cols; e.pitch = pl.pitch;
                    const long long rows = pl.n / pl.cols;
                    ranges.push_back({(uintptr_t)pl.w, (uintptr_t)pl.w + (size_t)((rows - 1) * pl.pitch + pl.cols) * 2, i, "plan operand"});
                    vec_ok = vec_ok && aligned(pl.w, 8) && pl.cols % 4 == 0 && pl.pitch % 4 == 0;
                }
            } else {
                PCNN_REQUIRE(pl.bias, PCNN_ERR_ARG, "%s: tensor %d: a bias for a plan created without one", fn, i);
                PCNN_REQUIRE(x.n == pl.K, PCNN_ERR_ARG, "%s: tensor %d: n = %ld, but the plan's bias has %d elements", fn, i, x.n, pl.K);
                e.mirror = pl.bias;
                ranges.push_back({(uintptr_t)pl.bias, (uintptr_t)pl.bias + (size_t)pl.K * sizeof(float), i, "plan bias"});
                vec_ok = vec_ok && aligned(pl.bias, 16);
            }
        }
        e.vec = vec_ok ? 1 : 0;
        chunks += (x.n + OPT_CHUNK - 1) / OPT_CHUNK;
        elements += x.n;
        state_floats += (x.n + 63) / 64 * 64;         // each tensor's state starts on a 256-byte boundary
    }
    PCNN_REQUIRE(chunks < (1LL << 31), PCNN_ERR_ARG, "%s: %lld chunks exceed the int range", fn, chunks);
    std::sort(ranges.begin(), ranges.end(), [](const Range &a, const Range &b) { return a.lo < b.lo; });
    for (size_t k = 1; k < ranges.size(); ++k)
        PCNN_REQUIRE(ranges[k].lo >= ranges[k - 1].hi, PCNN_ERR_ARG, "%s: overlapping buffers: the %s of tensor %d and the %s of tensor %d",
                     fn, ranges[k - 1].what, ranges[k - 1].tensor, ranges[k].what, ranges[k].tensor);

    pcnn_device_guard g(ctx->device);
    struct Guard {
        pcnn_optim *o;
        ~Guard() { free_optim(o); }
    } guard{new pcnn_optim()};
    pcnn_optim *o = guard.o;
    o->cfg = *cfg;
    o->count = count; o->nchunks = (int)chunks; o->elements = elements;
    const size_t nstate = (st0 ? 1 : 0) + (st1 ? 1 : 0);
    if (nstate) {
        PCNN_CUDA(cudaMalloc((void **)&o->d_state, (size_t)state_floats * nstate * sizeof(float)));
        PCNN_CUDA(cudaMemsetAsync(o->d_state, 0, (size_t)state_floats * nstate * sizeof(float), ctx->stream));
    }
    std::vector<int> chunk_tensor((size_t)chunks);
    long long soff = 0;
    for (int i = 0; i < count; ++i) {
        OptEntry &e = tab[i];
        if (st0) e.s0 = o->d_state + soff;
        if (st1) e.s1 = o->d_state + state_floats + soff;
        soff += (e.n + 63) / 64 * 64;
        const long long nc = (e.n + OPT_CHUNK - 1) / OPT_CHUNK;
        for (long long c = 0; c < nc; ++c) chunk_tensor[(size_t)(e.chunk0 + c)] = i;
        o->nvec += e.vec;
        if (t[i].plan_part == 1 && !e.dst) {
            o->toeplitz.push_back(t[i].plan);
            o->toeplitz_filt.push_back(t[i].param);
        }
    }
    PCNN_CUDA(cudaMalloc((void **)&o->d_tab, (size_t)count * sizeof(OptEntry)));
    PCNN_CUDA(cudaMalloc((void **)&o->d_chunks, (size_t)chunks * sizeof(int)));
    PCNN_CUDA(cudaMemcpyAsync(o->d_tab, tab.data(), (size_t)count * sizeof(OptEntry), cudaMemcpyHostToDevice, ctx->stream));
    PCNN_CUDA(cudaMemcpyAsync(o->d_chunks, chunk_tensor.data(), (size_t)chunks * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    PCNN_CUDA(cudaStreamSynchronize(ctx->stream));      // the host vectors go out of scope
    o->host = tab;
    const long long cap = (long long)ctx->sm_count * OPT_CTAS_PER_SM;
    o->grid = (int)(chunks < cap ? chunks : cap);
    guard.o = nullptr;
    *out = o;
    return PCNN_OK;
}

extern "C" int pcnn_optim_step(pcnn_ctx *ctx, pcnn_optim *o, float lr) {
    const char *fn = "pcnn_optim_step";
    PCNN_REQUIRE(ctx && o, PCNN_ERR_ARG, "%s: NULL context or optimizer", fn);
    PCNN_REQUIRE(!std::isnan(lr) && lr >= 0.0f, PCNN_ERR_ARG, "%s: lr %g: must be >= 0 and not NaN", fn, (double)lr);
    const pcnn_optim_config &c = o->cfg;
    const long long t = o->steps + 1;
    OptStep s{};
    s.neg_lr = -lr; s.lr = lr;
    s.mu = c.momentum; s.omega = (float)(1.0 - (double)c.dampening);
    s.momentum = c.momentum != 0.0f; s.first = t == 1;
    if (c.kind == PCNN_OPTIM_ADAMW) {
        s.a1 = (float)(1.0 - (double)c.beta1);
        s.beta2 = c.beta2;
        s.a2 = (float)(1.0 - (double)c.beta2);
        s.eps = c.eps;
        s.c2 = (float)std::sqrt(1.0 - std::pow((double)c.beta2, (double)t));
        s.neg_s = -(float)((double)lr / (1.0 - std::pow((double)c.beta1, (double)t)));
    }
    pcnn_device_guard g(ctx->device);
    const void *k = c.kind == PCNN_OPTIM_ADAMW ? (const void *)k_optim<PCNN_OPTIM_ADAMW, false>
                    : c.nesterov              ? (const void *)k_optim<PCNN_OPTIM_SGD, true>
                                              : (const void *)k_optim<PCNN_OPTIM_SGD, false>;
    void *args[] = {&o->d_tab, &o->d_chunks, &o->nchunks, &s};
    PCNN_CUDA(cudaLaunchKernel(k, dim3((unsigned)o->grid), dim3(OPT_THREADS), args, 0, ctx->stream));
    PCNN_CHECK_LAUNCH(ctx);
    for (size_t i = 0; i < o->toeplitz.size(); ++i) {
        const int rc = pcnn_conv_plan_set_params(ctx, o->toeplitz[i], o->toeplitz_filt[i], nullptr);
        if (rc) return rc;
    }
    o->steps = t;
    return PCNN_OK;
}

extern "C" int pcnn_optim_state(pcnn_optim *o, int i, float **state0_dev, float **state1_dev) {
    PCNN_REQUIRE(o && state0_dev && state1_dev, PCNN_ERR_ARG, "pcnn_optim_state: NULL argument");
    PCNN_REQUIRE(i >= 0 && i < o->count, PCNN_ERR_ARG, "pcnn_optim_state: tensor %d outside 0..%d", i, o->count - 1);
    *state0_dev = o->host[i].s0;
    *state1_dev = o->host[i].s1;
    return PCNN_OK;
}

extern "C" int pcnn_optim_info(pcnn_optim *o, long *out6) {
    PCNN_REQUIRE(o && out6, PCNN_ERR_ARG, "pcnn_optim_info: NULL argument");
    const long v[6] = {o->count, (long)o->elements, o->nvec, o->nchunks, o->grid, (long)o->steps};
    memcpy(out6, v, sizeof(v));
    return PCNN_OK;
}

extern "C" int pcnn_optim_destroy(pcnn_ctx *ctx, pcnn_optim *o) {
    PCNN_REQUIRE(ctx, PCNN_ERR_ARG, "pcnn_optim_destroy: ctx is NULL");
    if (!o) return PCNN_OK;
    pcnn_device_guard g(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    free_optim(o);
    return PCNN_OK;
}
