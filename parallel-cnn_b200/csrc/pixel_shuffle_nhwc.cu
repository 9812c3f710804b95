// parallel-cnn_b200/csrc/pixel_shuffle_nhwc.cu -- sub-pixel rearrangement between device-trained layers (pcnn_pixel_shuffle_nhwc_bf16,
// pcnn_pixel_unshuffle_nhwc_bf16 and the host-only pcnn_pixel_shuffle_info), as torch.nn.functional.pixel_shuffle / pixel_unshuffle
// written for dense NHWC bf16 maps.  With the coarse map [N][H][W][C r^2] and the fine map [N][H r][W r][C]:
//     fine[n][h r + i][w r + j][c] = coarse[n][h][w][c r^2 + i r + j]
// The shuffle writes the fine map from the coarse one, the unshuffle the coarse map from the fine one.  No arithmetic: every
// element is a 16-bit copy, so NaN payloads and -0 come through unchanged.
//
// One CTA per tile of P coarse pixels x a chunk of Cc fine channels.  On the coarse side a tile pixel is one contiguous run of
// Cc r^2 elements; on the fine side each of its r^2 fine pixels is a contiguous run of Cc channels, and for a fixed sub-row i the
// tile's consecutive coarse pixels of one image row cover a contiguous run of fine pixels.  So the tile goes through shared memory:
// the coarse side is read (or written) as it lies, the fine side in (i, pixel, j, channel) order, and the stride-r^2 gather
// happens in shared memory (tile_slot), never in global memory.  VEC = 8 moves 16 bytes per access (C % 8 == 0), VEC = 1 two bytes.
#include "pcnn_internal.h"

#include <cstdint>

namespace {

constexpr int PS_THREADS = 256;
constexpr int PS_TILE_ELEMS = 4096;          // elements of one tile
constexpr int PS_SMEM_ELEMS = PS_TILE_ELEMS + PS_TILE_ELEMS / 8;
constexpr int PS_MAX_R = 8;

// where tile element e lies in shared memory: 16 bytes of padding after every 128, so that the fine side's stride-r^2 gathers of
// neighbouring channel groups fall in different banks while a 16-byte run stays one aligned vector
__device__ __forceinline__ int tile_slot(int e) { return e + 8 * (e >> 6); }

// the coarse channel that holds fine channel c at sub-pixel (i, j), within a chunk of C fine channels
__device__ __forceinline__ int coarse_channel(int c, int i, int j, int r, int C) {
    return c * r * r + i * r + j;
}

struct PsArgs {
    const uint16_t *src;
    uint16_t *dst;
    int Hc, Wc, C, r;        // coarse height and width, fine channels, factor
    int P, Cc, chunks;       // coarse pixels per tile, fine channels per chunk, chunks per pixel block
    int M;                   // coarse pixels N Hc Wc
};

template <int VEC>
struct alignas(2 * VEC) U16Vec {
    uint16_t v[VEC];
};

// UNSHUFFLE false: src coarse, dst fine; true: src fine, dst coarse
template <int VEC, bool UNSHUFFLE>
__global__ void __launch_bounds__(PS_THREADS) k_pixel_shuffle(const PsArgs a) {
    __shared__ __align__(16) uint16_t tile[PS_SMEM_ELEMS];
    const int pb = blockIdx.x / a.chunks, cb = blockIdx.x % a.chunks;
    const int m0 = pb * a.P, np = min(a.P, a.M - m0);
    const int c0 = cb * a.Cc, cc = min(a.Cc, a.C - c0);
    const int r = a.r, r2 = r * r, L = cc * r2;          // tile elements per coarse pixel
    const int coarse_pitch = a.C * r2, Hf = a.Hc * r, Wf = a.Wc * r;
    using V = U16Vec<VEC>;

    // the coarse side: np runs of L elements, pixel m0 + p's run at (m0 + p) C r^2 + c0 r^2
    auto coarse = [&](bool load) {
        const int per = L / VEC;
#pragma unroll 4
        for (int v = threadIdx.x; v < np * per; v += PS_THREADS) {
            const int p = v / per, e = (v - p * per) * VEC;
            V *g = reinterpret_cast<V *>(const_cast<uint16_t *>(load ? a.src : a.dst) + (m0 + p) * coarse_pitch + c0 * r2 + e);
            V *s = reinterpret_cast<V *>(tile + tile_slot(p * L + e));
            if (load) *s = *g; else *g = *s;
        }
    };
    // the fine side, in (i, p, j, channel group) order: consecutive threads touch consecutive addresses along a fine row
    auto fine = [&](bool load) {
        const int G = cc / VEC;
#pragma unroll 2
        for (int v = threadIdx.x; v < r * np * r * G; v += PS_THREADS) {
            int t = v;
            const int g = t % G;
            t /= G;
            const int j = t % r;
            t /= r;
            const int p = t % np, i = t / np;
            const int m = m0 + p, w = m % a.Wc, hn = m / a.Wc, h = hn % a.Hc, n = hn / a.Hc;
            uint16_t *gp = const_cast<uint16_t *>(load ? a.src : a.dst) + (((n * Hf + h * r + i) * Wf + w * r + j) * a.C + c0 + g * VEC);
            if (load) {
                const V x = *reinterpret_cast<const V *>(gp);
#pragma unroll
                for (int k = 0; k < VEC; ++k) tile[tile_slot(p * L + coarse_channel(g * VEC + k, i, j, r, cc))] = x.v[k];
            } else {
                V y;
#pragma unroll
                for (int k = 0; k < VEC; ++k) y.v[k] = tile[tile_slot(p * L + coarse_channel(g * VEC + k, i, j, r, cc))];
                *reinterpret_cast<V *>(gp) = y;
            }
        }
    };
    if (UNSHUFFLE) {
        fine(true);
        __syncthreads();
        coarse(false);
    } else {
        coarse(true);
        __syncthreads();
        fine(false);
    }
}

struct PsShape {
    PsArgs a;
    int vec, grid;
};

// the shape rules of both directions; H, W, C are the op's own input: coarse [N][H][W][C r^2] for the shuffle, fine [N][H][W][C]
// for the unshuffle
int ps_shape(const char *fn, int N, int H, int W, int C, int r, bool unshuffle, PsShape *s) {
    PCNN_REQUIRE(N >= 1 && H >= 1 && W >= 1 && C >= 1, PCNN_ERR_ARG, "%s: N = %d, H = %d, W = %d, C = %d: each must be >= 1", fn, N, H,
                 W, C);
    PCNN_REQUIRE(r >= 1 && r <= PS_MAX_R, PCNN_ERR_ARG, "%s: r = %d: the factor must be 1 .. %d", fn, r, PS_MAX_R);
    PCNN_REQUIRE(!unshuffle || (H % r == 0 && W % r == 0), PCNN_ERR_ARG, "%s: H = %d, W = %d: both must be multiples of r = %d", fn, H,
                 W, r);
    const double elems = (double)N * H * W * C * (unshuffle ? 1.0 : (double)r * r);
    PCNN_REQUIRE(elems <= (double)INT32_MAX, PCNN_ERR_ARG, "%s: N H W C r^2 = %.0f elements: each map must hold at most 2^31 - 1", fn,
                 elems);
    const int r2 = r * r;
    PsArgs a;
    memset(&a, 0, sizeof(a));
    a.Hc = unshuffle ? H / r : H;
    a.Wc = unshuffle ? W / r : W;
    a.C = C;
    a.r = r;
    a.M = N * a.Hc * a.Wc;
    s->vec = C % 8 == 0 ? 8 : 1;
    a.Cc = C * r2 <= PS_TILE_ELEMS ? C : PS_TILE_ELEMS / r2 / s->vec * s->vec;
    a.chunks = (C + a.Cc - 1) / a.Cc;
    a.P = PS_TILE_ELEMS / (a.Cc * r2);
    s->grid = (a.M + a.P - 1) / a.P * a.chunks;
    s->a = a;
    return PCNN_OK;
}

int ps_run(const char *fn, pcnn_ctx *ctx, const void *x, void *y, int N, int H, int W, int C, int r, bool unshuffle) {
    PCNN_REQUIRE(ctx && x && y, PCNN_ERR_ARG, "%s: NULL argument", fn);
    PsShape s;
    const int rc = ps_shape(fn, N, H, W, C, r, unshuffle, &s);
    if (rc) return rc;
    PCNN_REQUIRE((((uintptr_t)x | (uintptr_t)y) & 15) == 0, PCNN_ERR_ARG, "%s: x and y must be 16-byte aligned", fn);
    const size_t bytes = (size_t)N * H * W * C * 2 * (unshuffle ? 1 : r * r);
    const uintptr_t px = (uintptr_t)x, py = (uintptr_t)y;
    PCNN_REQUIRE(px + bytes <= py || py + bytes <= px, PCNN_ERR_ARG, "%s: x and y overlap: a permutation cannot run in place", fn);
    pcnn_device_guard g(ctx->device);
    PsArgs a = s.a;
    a.src = static_cast<const uint16_t *>(x);
    a.dst = static_cast<uint16_t *>(y);
    if (unshuffle) {
        if (s.vec == 8) k_pixel_shuffle<8, true><<<s.grid, PS_THREADS, 0, ctx->stream>>>(a);
        else k_pixel_shuffle<1, true><<<s.grid, PS_THREADS, 0, ctx->stream>>>(a);
    } else {
        if (s.vec == 8) k_pixel_shuffle<8, false><<<s.grid, PS_THREADS, 0, ctx->stream>>>(a);
        else k_pixel_shuffle<1, false><<<s.grid, PS_THREADS, 0, ctx->stream>>>(a);
    }
    PCNN_CHECK_LAUNCH(ctx);
    return PCNN_OK;
}

}  // namespace

extern "C" int pcnn_pixel_shuffle_info(int N, int H, int W, int C, int r, int unshuffle, long long *out6) {
    const char *fn = "pcnn_pixel_shuffle_info";
    PCNN_REQUIRE(out6, PCNN_ERR_ARG, "%s: NULL out6", fn);
    PCNN_REQUIRE(unshuffle == 0 || unshuffle == 1, PCNN_ERR_ARG, "%s: unshuffle = %d: 0 or 1 is required", fn, unshuffle);
    PsShape s;
    const int rc = ps_shape(fn, N, H, W, C, r, unshuffle != 0, &s);
    if (rc) return rc;
    out6[0] = s.vec;
    out6[1] = s.grid;
    out6[2] = PS_THREADS;
    out6[3] = PS_SMEM_ELEMS * 2;
    out6[4] = s.a.P;
    out6[5] = s.a.Cc;
    return PCNN_OK;
}

extern "C" int pcnn_pixel_shuffle_nhwc_bf16(pcnn_ctx *ctx, const void *x_bf16_dev, void *y_bf16_dev, int N, int H, int W, int C, int r) {
    return ps_run("pcnn_pixel_shuffle_nhwc_bf16", ctx, x_bf16_dev, y_bf16_dev, N, H, W, C, r, false);
}

extern "C" int pcnn_pixel_unshuffle_nhwc_bf16(pcnn_ctx *ctx, const void *x_bf16_dev, void *y_bf16_dev, int N, int H, int W, int C, int r) {
    return ps_run("pcnn_pixel_unshuffle_nhwc_bf16", ctx, x_bf16_dev, y_bf16_dev, N, H, W, C, r, true);
}
