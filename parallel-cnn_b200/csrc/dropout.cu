// parallel-cnn_b200/csrc/dropout.cu -- dropout and stochastic depth (drop path) of bf16 rows (pcnn_dropout_bf16): y = x * m (+ r),
// m = 0 for a dropped element and 1 / (1 - p) for a kept one, the mask drawn from Philox4x32-10 at an index that depends on the
// element (element mode) or on the row (per-sample mode) alone.  The backward is the same call on dy with the forward's (seed,
// call, p, mode) and no r.  The contract, every operation in its order, is in include/pcnn.h.
//
// The pass is elementwise and HBM-bound but for the generator: with row_elems % 8 == 0 and row_pitch % 8 == 0 a thread moves
// 16-byte vectors of 8 elements of one row (two Philox calls in element mode, one in per-sample mode), otherwise single elements.
// A grid-stride loop whose grid is a function of the shape alone walks the vectors; which thread handles an element never
// changes a bit, since the draw is a function of (seed, call, index).  p = 0 takes a kernel without the generator.
#include "pcnn_internal.h"
#include "philox.cuh"

#include <cuda_bf16.h>

#include <algorithm>
#include <cmath>

namespace {

constexpr int DROP_THREADS = 256;
constexpr long long DROP_MAX_GRID = 1056;   // most CTAs of the grid-stride loop: 8 of 256 threads (<= 32 registers) on each of 132 SMs
enum { MODE_KEEP = 0, MODE_ELEMENT = 1, MODE_SAMPLE = 2 };

template <int VEC>
struct alignas(2 * VEC) BfVec {
    __nv_bfloat16 h[VEC];
};

struct DropArgs {
    long long N;
    int row_elems, row_pitch;   // elements; row_pitch >= row_elems
    int vpr;                    // vectors per row (row_elems / VEC)
    long long sq;               // the grid stride in vectors, as whole rows (sq) and the remainder (sr < vpr)
    int sr;
    unsigned T;                 // dropped iff draw < T
    float scale;
    unsigned k0, k1, c2, c3;    // the Philox key (seed lo, hi) and the counter's upper words (call lo, hi)
};

// word (i & 3) of the block of counter (i >> 2, call)
__device__ __forceinline__ unsigned draw(unsigned long long i, const DropArgs &a) {
    const unsigned long long q = i >> 2;
    const uint4 w = philox4x32_10((unsigned)q, (unsigned)(q >> 32), a.c2, a.c3, a.k0, a.k1);
    const unsigned j = (unsigned)i & 3;
    return j == 0 ? w.x : j == 1 ? w.y : j == 2 ? w.z : w.w;
}

__device__ __forceinline__ float keep_scale(unsigned d, const DropArgs &a) { return d < a.T ? 0.0f : a.scale; }

// y = bf16_rn(float(x) * m), or bf16_rn(float(r) + RN(float(x) * m)) with r.  x, r and y may be the same buffer: each element is
// read, then written, by one thread.
template <int VEC, int MODE>
__global__ void __launch_bounds__(DROP_THREADS) k_dropout(const __nv_bfloat16 *x, const __nv_bfloat16 *r, __nv_bfloat16 *y, DropArgs a) {
    const unsigned v0 = blockIdx.x * DROP_THREADS + threadIdx.x;
    long long n = v0 / (unsigned)a.vpr;
    int jv = (int)(v0 - (unsigned)n * (unsigned)a.vpr);
    for (; n < a.N; n += a.sq, jv += a.sr) {
        if (jv >= a.vpr) {
            jv -= a.vpr;
            if (++n >= a.N) break;
        }
        const long long off = n * a.row_pitch + (long long)jv * VEC;
        const BfVec<VEC> xv = *reinterpret_cast<const BfVec<VEC> *>(x + off);
        BfVec<VEC> rv;
        if (r) rv = *reinterpret_cast<const BfVec<VEC> *>(r + off);
        float m[VEC];
        if (MODE == MODE_KEEP) {
#pragma unroll
            for (int c = 0; c < VEC; ++c) m[c] = a.scale;
        } else if (MODE == MODE_SAMPLE) {
            const float s = keep_scale(draw((unsigned long long)n, a), a);
#pragma unroll
            for (int c = 0; c < VEC; ++c) m[c] = s;
        } else if (VEC == 8) {     // i = n row_elems + 8 jv is a multiple of 8: the eight words of counters i / 4 and i / 4 + 1
            const unsigned long long q = ((unsigned long long)n * a.row_elems + 8ull * jv) >> 2;
            const uint4 w0 = philox4x32_10((unsigned)q, (unsigned)(q >> 32), a.c2, a.c3, a.k0, a.k1);
            const uint4 w1 = philox4x32_10((unsigned)(q + 1), (unsigned)((q + 1) >> 32), a.c2, a.c3, a.k0, a.k1);
            const unsigned d[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
            for (int c = 0; c < VEC; ++c) m[c] = keep_scale(d[c], a);
        } else {
            m[0] = keep_scale(draw((unsigned long long)n * a.row_elems + jv, a), a);
        }
        BfVec<VEC> out;
#pragma unroll
        for (int c = 0; c < VEC; ++c) {
            float v = __fmul_rn(__bfloat162float(xv.h[c]), m[c]);
            if (r) v = __fadd_rn(__bfloat162float(rv.h[c]), v);
            out.h[c] = __float2bfloat16_rn(v);
        }
        *reinterpret_cast<BfVec<VEC> *>(y + off) = out;
    }
}

typedef void (*drop_fn)(const __nv_bfloat16 *, const __nv_bfloat16 *, __nv_bfloat16 *, DropArgs);

struct DropShape {
    DropArgs a;
    int vec, grid;
    long long per_thread;   // elements of the busiest thread
};

// the domain, one message per rule, and the launch: a function of (N, row_elems, row_pitch, p, per_sample) alone
int drop_shape(const char *fn, int N, int row_elems, int row_pitch, double p, int per_sample, DropShape *s) {
    PCNN_REQUIRE(N >= 1 && row_elems >= 1, PCNN_ERR_ARG, "%s: N = %d, row_elems = %d: each must be >= 1", fn, N, row_elems);
    const int pitch = row_pitch == 0 ? row_elems : row_pitch;
    PCNN_REQUIRE(pitch >= row_elems, PCNN_ERR_ARG, "%s: row_pitch = %d: 0 (dense) or >= row_elems = %d is required", fn, row_pitch,
                 row_elems);
    PCNN_REQUIRE(std::isfinite(p) && p >= 0.0 && p < 1.0, PCNN_ERR_ARG, "%s: p = %g: a finite p with 0 <= p < 1 is required", fn, p);
    PCNN_REQUIRE(per_sample == 0 || per_sample == 1, PCNN_ERR_ARG, "%s: per_sample = %d: 0 (element) or 1 (per sample) is required", fn,
                 per_sample);
    DropArgs &a = s->a;
    a.N = N;
    a.row_elems = row_elems;
    a.row_pitch = pitch;
    s->vec = row_elems % 8 == 0 && pitch % 8 == 0 ? 8 : 1;
    a.vpr = row_elems / s->vec;
    const long long total = (long long)N * a.vpr;
    s->grid = (int)std::min(DROP_MAX_GRID, (total + DROP_THREADS - 1) / DROP_THREADS);
    const long long stride = (long long)s->grid * DROP_THREADS;
    a.sq = stride / a.vpr;
    a.sr = (int)(stride % a.vpr);
    s->per_thread = (total + stride - 1) / stride * s->vec;
    const double t = std::nearbyint(p * 4294967296.0);        // p 2^32 is exact in double; ties to even
    a.T = t >= 4294967295.0 ? 0xFFFFFFFFu : (unsigned)t;     // the uint32 nearest to p 2^32
    a.scale = (float)(1.0 / (1.0 - p));
    return PCNN_OK;
}

bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// two buffers of `bytes` each are the same buffer or share no byte
bool same_or_disjoint(const void *a, const void *b, size_t bytes) {
    if (!a || !b || a == b) return true;
    const uintptr_t pa = (uintptr_t)a, pb = (uintptr_t)b;
    return pa + bytes <= pb || pb + bytes <= pa;
}

}  // namespace

extern "C" int pcnn_dropout_bf16_info(int N, int row_elems, int row_pitch, double p, int per_sample, long long *out5) {
    const char *fn = "pcnn_dropout_bf16_info";
    PCNN_REQUIRE(out5, PCNN_ERR_ARG, "%s: NULL out5", fn);
    DropShape s;
    const int rc = drop_shape(fn, N, row_elems, row_pitch, p, per_sample, &s);
    if (rc) return rc;
    unsigned scale_bits;
    memcpy(&scale_bits, &s.a.scale, 4);
    out5[0] = s.a.T;
    out5[1] = scale_bits;
    out5[2] = s.vec;
    out5[3] = s.grid;
    out5[4] = s.per_thread;
    return PCNN_OK;
}

extern "C" int pcnn_dropout_bf16(pcnn_ctx *ctx, const void *x_bf16, const void *r_bf16, void *y_bf16, int N, int row_elems, int row_pitch,
                                 double p, int per_sample, unsigned long long seed, unsigned long long call) {
    const char *fn = "pcnn_dropout_bf16";
    PCNN_REQUIRE(ctx && x_bf16 && y_bf16, PCNN_ERR_ARG, "%s: NULL context, x or y (only r may be NULL)", fn);
    DropShape s;
    int rc = drop_shape(fn, N, row_elems, row_pitch, p, per_sample, &s);
    if (rc) return rc;
    PCNN_REQUIRE(aligned16(x_bf16) && aligned16(r_bf16) && aligned16(y_bf16), PCNN_ERR_ARG, "%s: x, r and y must be 16-byte aligned", fn);
    const size_t bytes = ((size_t)(N - 1) * s.a.row_pitch + s.a.row_elems) * 2;
    PCNN_REQUIRE(same_or_disjoint(x_bf16, r_bf16, bytes) && same_or_disjoint(x_bf16, y_bf16, bytes) &&
                     same_or_disjoint(r_bf16, y_bf16, bytes),
                 PCNN_ERR_ARG, "%s: overlapping buffers: x, r and y must each be the same buffer or share no byte", fn);
    s.a.k0 = (unsigned)seed;
    s.a.k1 = (unsigned)(seed >> 32);
    s.a.c2 = (unsigned)call;
    s.a.c3 = (unsigned)(call >> 32);
    pcnn_device_guard dg(ctx->device);
    const int mode = s.a.T == 0 ? MODE_KEEP : per_sample ? MODE_SAMPLE : MODE_ELEMENT;
    static const drop_fn table[2][3] = {{k_dropout<1, MODE_KEEP>, k_dropout<1, MODE_ELEMENT>, k_dropout<1, MODE_SAMPLE>},
                                        {k_dropout<8, MODE_KEEP>, k_dropout<8, MODE_ELEMENT>, k_dropout<8, MODE_SAMPLE>}};
    table[s.vec == 8][mode]<<<s.grid, DROP_THREADS, 0, ctx->stream>>>(static_cast<const __nv_bfloat16 *>(x_bf16),
                                                                       static_cast<const __nv_bfloat16 *>(r_bf16),
                                                                       static_cast<__nv_bfloat16 *>(y_bf16), s.a);
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}
