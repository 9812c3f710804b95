// parallel-cnn_b200/csrc/gaussian_latent.cu -- the reparameterized Gaussian latent of a variational autoencoder
// (pcnn_gaussian_latent_bf16_fwd / _bwd): z = mu + exp(lv / 2) eps with eps a standard normal drawn by Philox4x32-10 and
// Box-Muller, the KL divergence of each row from N(0, I), and the gradients of both.  The fp32 operations and their order are
// include/pcnn.h's.
//
// stats is R rows of ld bf16 elements, mu in columns 0 .. L-1 and logvar in L .. 2L-1: a LinearLayer's output with O = 2L, read in
// place.  Nothing is stored between the passes: the backward draws eps again from (seed, call, r L + j).  One CTA per tile of
// GL_TILE rows, walking the columns in chunks of GL_CHUNK: each thread takes VEC consecutive columns of one row (VEC = 8, 16-byte
// accesses, when L, ld and ldz are multiples of 8) and leaves their KL terms in shared memory; one thread per row then adds them
// in ascending column order.  No atomics: a row's bits depend on (seed, call, r, L) alone.
#include "pcnn_internal.h"
#include "philox.cuh"

#include <cuda_bf16.h>

#include <cmath>

namespace {

constexpr int GL_THREADS = 256;
constexpr int GL_TILE = 64;                   // rows per CTA
constexpr int GL_CHUNK = 128;                 // columns per pass over shared memory (a multiple of 8)
constexpr unsigned GL_DOMAIN = 0xE0000000u;   // word 1 of every latent counter (include/pcnn.h: no other draw reaches it)

struct GlArgs {
    const __nv_bfloat16 *stats, *dz;
    __nv_bfloat16 *z, *dstats;
    float *kl;
    int R, L, ld, ldz;
    unsigned k0, k1, c2, c3;                  // key (seed lo, hi), counter words 2 and 3 (call lo, hi)
    float kl_scale;
};

template <int VEC>
struct alignas(2 * VEC) Bf16Vec {
    __nv_bfloat16 v[VEC];
};

// the Box-Muller pair of words (wa, wb): rad cos and rad sin of 2 pi u2, rad = sqrt(-2 log u1)
__device__ __forceinline__ void box_muller(unsigned wa, unsigned wb, float *n0, float *n1) {
    const float u1 = __fmul_rn((float)((wa >> 8) + 1u), __int_as_float(0x33800000));       // 2^-24, exact
    const float rad = __fsqrt_rn(__fmul_rn(-2.0f, log1p_f32(__fsub_rn(u1, 1.0f))));
    float sn, cs;
    sincos_2pi_f32(wb >> 8, &sn, &cs);
    *n0 = __fmul_rn(rad, cs);
    *n1 = __fmul_rn(rad, sn);
}

__device__ __forceinline__ uint4 gl_block(const GlArgs &a, unsigned long long q) {
    return philox4x32_10((unsigned)q, GL_DOMAIN | (unsigned)(q >> 32), a.c2, a.c3, a.k0, a.k1);
}

// eps of elements i .. i + VEC - 1 (i a multiple of VEC): two whole blocks for VEC = 8, one Box-Muller pair for VEC = 1
template <int VEC>
__device__ __forceinline__ void draw(const GlArgs &a, unsigned long long i, float (&e)[VEC]) {
    if constexpr (VEC == 8) {
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const uint4 w = gl_block(a, (i >> 2) + b);
            box_muller(w.x, w.y, &e[4 * b], &e[4 * b + 1]);
            box_muller(w.z, w.w, &e[4 * b + 2], &e[4 * b + 3]);
        }
    } else {
        const uint4 w = gl_block(a, i >> 2);
        const bool hi = (i >> 1) & 1;
        float n0, n1;
        box_muller(hi ? w.z : w.x, hi ? w.w : w.y, &n0, &n1);
        e[0] = (i & 1) ? n1 : n0;
    }
}

template <int VEC, bool TRAIN>
__global__ void __launch_bounds__(GL_THREADS) k_gaussian_latent_fwd(const GlArgs a) {
    __shared__ float terms[GL_TILE][GL_CHUNK + 1];
    const int r0 = blockIdx.x * GL_TILE;
    const int nr = min(GL_TILE, a.R - r0);
    float s = 0.0f;                                          // thread p < nr: the running KL sum of row r0 + p
    for (int c0 = 0; c0 < a.L; c0 += GL_CHUNK) {
        const int cc = min(GL_CHUNK, a.L - c0), G = cc / VEC;
        for (int v = threadIdx.x; v < nr * G; v += GL_THREADS) {
            const int p = v / G, cl = (v - p * G) * VEC;
            const long long r = r0 + p;
            const int j = c0 + cl;
            const Bf16Vec<VEC> mv = *reinterpret_cast<const Bf16Vec<VEC> *>(a.stats + r * a.ld + j);
            const Bf16Vec<VEC> lv = *reinterpret_cast<const Bf16Vec<VEC> *>(a.stats + r * a.ld + a.L + j);
            Bf16Vec<VEC> zv;
            float e[VEC];
            if constexpr (TRAIN) draw<VEC>(a, (unsigned long long)r * a.L + j, e);
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                const float mu = __bfloat162float(mv.v[k]), l = __bfloat162float(lv.v[k]);
                if constexpr (TRAIN)
                    zv.v[k] = __float2bfloat16_rn(__fadd_rn(mu, __fmul_rn(exp_f32(__fmul_rn(0.5f, l)), e[k])));
                else
                    zv.v[k] = mv.v[k];
                if (a.kl) terms[p][cl + k] = __fsub_rn(__fsub_rn(__fadd_rn(__fmul_rn(mu, mu), exp_f32(l)), 1.0f), l);
            }
            *reinterpret_cast<Bf16Vec<VEC> *>(a.z + r * a.ldz + j) = zv;
        }
        if (a.kl) {
            __syncthreads();
            if (threadIdx.x < nr)
                for (int c = 0; c < cc; ++c) s = __fadd_rn(s, terms[threadIdx.x][c]);
            __syncthreads();
        }
    }
    if (a.kl && threadIdx.x < nr) a.kl[r0 + threadIdx.x] = __fmul_rn(0.5f, s);
}

template <int VEC>
__global__ void __launch_bounds__(GL_THREADS) k_gaussian_latent_bwd(const GlArgs a) {
    const int r0 = blockIdx.x * GL_TILE;
    const int nr = min(GL_TILE, a.R - r0), G = a.L / VEC;
    const float kh = __fmul_rn(a.kl_scale, 0.5f);
    for (int v = threadIdx.x; v < nr * G; v += GL_THREADS) {
        const int p = v / G, j = (v - p * G) * VEC;
        const long long r = r0 + p;
        const Bf16Vec<VEC> mv = *reinterpret_cast<const Bf16Vec<VEC> *>(a.stats + r * a.ld + j);
        const Bf16Vec<VEC> lv = *reinterpret_cast<const Bf16Vec<VEC> *>(a.stats + r * a.ld + a.L + j);
        const Bf16Vec<VEC> gv = *reinterpret_cast<const Bf16Vec<VEC> *>(a.dz + r * a.ldz + j);
        float e[VEC];
        draw<VEC>(a, (unsigned long long)r * a.L + j, e);
        Bf16Vec<VEC> dm, dl;
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            const float mu = __bfloat162float(mv.v[k]), l = __bfloat162float(lv.v[k]), g = __bfloat162float(gv.v[k]);
            dm.v[k] = __float2bfloat16_rn(__fadd_rn(g, __fmul_rn(a.kl_scale, mu)));
            const float t = __fmul_rn(__fmul_rn(__fmul_rn(0.5f, g), e[k]), exp_f32(__fmul_rn(0.5f, l)));
            dl.v[k] = __float2bfloat16_rn(__fadd_rn(t, __fmul_rn(kh, __fsub_rn(exp_f32(l), 1.0f))));
        }
        *reinterpret_cast<Bf16Vec<VEC> *>(a.dstats + r * a.ld + j) = dm;
        *reinterpret_cast<Bf16Vec<VEC> *>(a.dstats + r * a.ld + a.L + j) = dl;
    }
}

bool gl_disjoint(const void *a, size_t abytes, const void *b, size_t bbytes) {
    const uintptr_t pa = (uintptr_t)a, pb = (uintptr_t)b;
    return pa + abytes <= pb || pb + bbytes <= pa;
}

int gl_shape(const char *fn, int R, int L, int ld, int ldz) {
    PCNN_REQUIRE(R >= 1, PCNN_ERR_ARG, "%s: R = %d: at least 1 row is required", fn, R);
    PCNN_REQUIRE(L >= 1 && L <= 4096, PCNN_ERR_ARG, "%s: L = %d: 1 <= L <= 4096 is required", fn, L);
    PCNN_REQUIRE(ld >= 2 * L, PCNN_ERR_ARG, "%s: ld = %d, L = %d: ld >= 2 L is required", fn, ld, L);
    PCNN_REQUIRE(ldz >= L, PCNN_ERR_ARG, "%s: ldz = %d, L = %d: ldz >= L is required", fn, ldz, L);
    return PCNN_OK;
}

int gl_vec(int L, int ld, int ldz) { return (L % 8 == 0 && ld % 8 == 0 && ldz % 8 == 0) ? 8 : 1; }

GlArgs gl_args(int R, int L, int ld, int ldz, unsigned long long seed, unsigned long long call) {
    GlArgs a{};
    a.R = R;
    a.L = L;
    a.ld = ld;
    a.ldz = ldz;
    a.k0 = (unsigned)seed;
    a.k1 = (unsigned)(seed >> 32);
    a.c2 = (unsigned)call;
    a.c3 = (unsigned)(call >> 32);
    return a;
}

unsigned gl_grid(int R) { return (unsigned)((R + GL_TILE - 1) / GL_TILE); }

}  // namespace

extern "C" int pcnn_gaussian_latent_info(int R, int L, int ld, int ldz, long long *out6) {
    const char *fn = "pcnn_gaussian_latent_info";
    PCNN_REQUIRE(out6, PCNN_ERR_ARG, "%s: NULL argument", fn);
    const int rc = gl_shape(fn, R, L, ld, ldz);
    if (rc != PCNN_OK) return rc;
    out6[0] = gl_vec(L, ld, ldz);
    out6[1] = gl_grid(R);
    out6[2] = GL_THREADS;
    out6[3] = (long long)sizeof(float) * GL_TILE * (GL_CHUNK + 1);
    out6[4] = GL_TILE;
    out6[5] = GL_CHUNK;
    return PCNN_OK;
}

extern "C" int pcnn_gaussian_latent_bf16_fwd(pcnn_ctx *ctx, const void *stats_bf16_dev, int ld, void *z_bf16_dev, int ldz,
                                             float *kl_f32_dev, int R, int L, unsigned long long seed, unsigned long long call,
                                             int training) {
    const char *fn = "pcnn_gaussian_latent_bf16_fwd";
    PCNN_REQUIRE(ctx && stats_bf16_dev && z_bf16_dev, PCNN_ERR_ARG, "%s: NULL argument", fn);
    int rc = gl_shape(fn, R, L, ld, ldz);
    if (rc != PCNN_OK) return rc;
    PCNN_REQUIRE(training == 0 || training == 1, PCNN_ERR_ARG, "%s: training = %d is not 0 or 1", fn, training);
    PCNN_REQUIRE(!training || call >= 1, PCNN_ERR_ARG, "%s: call = 0: a training draw needs call >= 1", fn);
    PCNN_REQUIRE((((uintptr_t)stats_bf16_dev | (uintptr_t)z_bf16_dev | (uintptr_t)kl_f32_dev) & 15) == 0, PCNN_ERR_ARG,
                 "%s: stats, z and kl must be 16-byte aligned", fn);
    const size_t sbytes = ((size_t)(R - 1) * ld + 2 * L) * 2, zbytes = ((size_t)(R - 1) * ldz + L) * 2, kbytes = (size_t)R * 4;
    PCNN_REQUIRE((z_bf16_dev == stats_bf16_dev && ldz == ld) || gl_disjoint(z_bf16_dev, zbytes, stats_bf16_dev, sbytes), PCNN_ERR_ARG,
                 "%s: z overlaps stats without being stats at ldz == ld: only that in-place form is allowed", fn);
    PCNN_REQUIRE(!kl_f32_dev || (gl_disjoint(kl_f32_dev, kbytes, stats_bf16_dev, sbytes) &&
                                 gl_disjoint(kl_f32_dev, kbytes, z_bf16_dev, zbytes)),
                 PCNN_ERR_ARG, "%s: kl overlaps stats or z", fn);
    pcnn_device_guard g(ctx->device);
    GlArgs a = gl_args(R, L, ld, ldz, seed, call);
    a.stats = static_cast<const __nv_bfloat16 *>(stats_bf16_dev);
    a.z = static_cast<__nv_bfloat16 *>(z_bf16_dev);
    a.kl = kl_f32_dev;
    const unsigned grid = gl_grid(R);
    const bool v8 = gl_vec(L, ld, ldz) == 8;
    if (training) {
        if (v8) k_gaussian_latent_fwd<8, true><<<grid, GL_THREADS, 0, ctx->stream>>>(a);
        else k_gaussian_latent_fwd<1, true><<<grid, GL_THREADS, 0, ctx->stream>>>(a);
    } else {
        if (v8) k_gaussian_latent_fwd<8, false><<<grid, GL_THREADS, 0, ctx->stream>>>(a);
        else k_gaussian_latent_fwd<1, false><<<grid, GL_THREADS, 0, ctx->stream>>>(a);
    }
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

extern "C" int pcnn_gaussian_latent_bf16_bwd(pcnn_ctx *ctx, const void *stats_bf16_dev, int ld, const void *dz_bf16_dev, int ldz,
                                             void *dstats_bf16_dev, int R, int L, unsigned long long seed, unsigned long long call,
                                             float kl_scale) {
    const char *fn = "pcnn_gaussian_latent_bf16_bwd";
    PCNN_REQUIRE(ctx && stats_bf16_dev && dz_bf16_dev && dstats_bf16_dev, PCNN_ERR_ARG, "%s: NULL argument", fn);
    int rc = gl_shape(fn, R, L, ld, ldz);
    if (rc != PCNN_OK) return rc;
    PCNN_REQUIRE(call >= 1, PCNN_ERR_ARG, "%s: call = 0: the backward replays a training draw, which has call >= 1", fn);
    PCNN_REQUIRE(std::isfinite(kl_scale), PCNN_ERR_ARG, "%s: kl_scale = %g: a finite kl_scale is required", fn, (double)kl_scale);
    PCNN_REQUIRE((((uintptr_t)stats_bf16_dev | (uintptr_t)dz_bf16_dev | (uintptr_t)dstats_bf16_dev) & 15) == 0, PCNN_ERR_ARG,
                 "%s: stats, dz and dstats must be 16-byte aligned", fn);
    const size_t sbytes = ((size_t)(R - 1) * ld + 2 * L) * 2, zbytes = ((size_t)(R - 1) * ldz + L) * 2;
    PCNN_REQUIRE(dstats_bf16_dev == stats_bf16_dev || gl_disjoint(dstats_bf16_dev, sbytes, stats_bf16_dev, sbytes), PCNN_ERR_ARG,
                 "%s: dstats overlaps stats without being stats: only dstats == stats (in place) is allowed", fn);
    PCNN_REQUIRE(gl_disjoint(dstats_bf16_dev, sbytes, dz_bf16_dev, zbytes), PCNN_ERR_ARG, "%s: dstats overlaps dz", fn);
    pcnn_device_guard g(ctx->device);
    GlArgs a = gl_args(R, L, ld, ldz, seed, call);
    a.stats = static_cast<const __nv_bfloat16 *>(stats_bf16_dev);
    a.dz = static_cast<const __nv_bfloat16 *>(dz_bf16_dev);
    a.dstats = static_cast<__nv_bfloat16 *>(dstats_bf16_dev);
    a.kl_scale = kl_scale;
    const unsigned grid = gl_grid(R);
    if (gl_vec(L, ld, ldz) == 8) k_gaussian_latent_bwd<8><<<grid, GL_THREADS, 0, ctx->stream>>>(a);
    else k_gaussian_latent_bwd<1><<<grid, GL_THREADS, 0, ctx->stream>>>(a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
