"""Grid rules of the LeNet kernels that cap their grid and loop over the rest of the work, copied from their launchers, and
the batch sizes tests/test_laps_gpu.py runs them at.

  evaluation pass   k_fused<*, false>      a CTA takes images b, b + grid, ...         (pcnn_forward_batch, pcnn_test)
  LeNet-5 variant   k_l5_step<true/false>  a CTA takes images b, b + grid, ...         (pcnn_l5_*)
  operator tier     ops_kernels.cu         a thread takes items i, i + grid·threads, ... (the batched pcnn_* operators)
  planar ext ops    ext_kernels.cu         a thread (warp for softmax) does the same    (pcnn_maxpool_*, pcnn_softmax_ce)

Every batch size below is derived from these rules so that the loop runs at least twice on the device at hand.  SOURCE pins
each copied line to its text in the CUDA sources: a change to a rule fails tests/test_laps_cpu.py instead of quietly
taking the GPU tests back to one lap."""
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "parallel-cnn_b200", "csrc")
NB = 1024                       # golden training digits; larger batches tile them

# (file under csrc/, 1-based line, text that line contains)
SOURCE = [
    ("pcnn_internal.h", 24, "constexpr int FUSED_CTAS_PER_SM = 2;"),
    ("pcnn_internal.h", 27, "constexpr int MAX_SLOTS = 148 * 4;"),
    ("fused_kernels.cu", 67, "for (int b = b0; b < nb; b += gridDim.x, ++li) {"),
    ("fused_kernels.cu", 171, "int cap = ctx->sm_count * FUSED_CTAS_PER_SM;"),
    ("fused_kernels.cu", 172, "if (cap > MAX_SLOTS) cap = MAX_SLOTS;"),
    ("fused_kernels.cu", 173, "return B < cap ? B : cap;"),
    ("fused_kernels.cu", 797, "return launch_fused<false>(ctx, a, pixel_type, fused_grid(ctx, B));"),
    ("fused_kernels.cu", 815, "int rc = launch_fused<false>(ctx, a, s.pixel_type, fused_grid(ctx, (int)s.n));"),
    ("lenet5_kernels.cu", 81, "for (int b = blockIdx.x; b < a.B; b += gridDim.x) {"),
    ("lenet5_kernels.cu", 413, "const int cap = ctx->sm_count * 2;"),
    ("lenet5_kernels.cu", 414, "return B < cap ? B : cap;"),
    ("lenet5_kernels.cu", 433, "const int grid = l5_grid(ctx, B);"),
    ("lenet5_kernels.cu", 464, "return l5_launch<false>(ctx, a, l5_grid(ctx, B));"),
    ("ops_kernels.cu", 29, "long b = (n + threads - 1) / threads;"),
    ("ops_kernels.cu", 30, "if (b < 1) b = 1;"),
    ("ops_kernels.cu", 31, "if (b > 148L * 32) b = 148L * 32;"),
    ("ops_kernels.cu", 35, "#define GRID_STRIDE(i, n) for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < (n); "
                           "i += (long)gridDim.x * blockDim.x)"),
    ("ext_kernels.cu", 12, "long b = (items + threads - 1) / threads;"),
    ("ext_kernels.cu", 13, "long cap = (long)ctx->sm_count * 8;"),
    ("ext_kernels.cu", 14, "if (b > cap) b = cap;"),
    ("ext_kernels.cu", 15, "return (int)(b < 1 ? 1 : b);"),
    ("ext_kernels.cu", 27, "for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {"),
    ("ext_kernels.cu", 61, "for (long idx = blockIdx.x * (long)blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {"),
    ("ext_kernels.cu", 81, "const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;"),
    ("ext_kernels.cu", 107, "const long total = (long)planes * (H / k) * (W / k);"),
    ("ext_kernels.cu", 108, "const int grid = grid_for(ctx, total, 256);"),
    ("ext_kernels.cu", 120, "const long total = (long)planes * H * W;"),
    ("ext_kernels.cu", 121, "k_maxpool_bwd<<<grid_for(ctx, total, 256), 256, 0, ctx->stream>>>"),
    ("ext_kernels.cu", 131, "k_softmax_ce<<<grid_for(ctx, (long)B * 32, 256), 256, 0, ctx->stream>>>"),
]

# ---------------------------------------------------------------- evaluation pass and LeNet-5 variant: images per CTA
FUSED_CTAS_PER_SM = 2           # pcnn_internal.h:24
MAX_SLOTS = 148 * 4             # pcnn_internal.h:27


def fused_grid(sm_count, B):
    """fused_kernels.cu:170-174 (fused_grid), the grid of pcnn_forward_batch (:797) and pcnn_test (:815)"""
    cap = sm_count * FUSED_CTAS_PER_SM
    if cap > MAX_SLOTS:
        cap = MAX_SLOTS
    return B if B < cap else cap


def l5_grid(sm_count, B):
    """lenet5_kernels.cu:412-415 (l5_grid), the grid of every pcnn_l5_* launch (:433, :464)"""
    cap = sm_count * 2
    return B if B < cap else cap


def images_per_cta(B, grid):
    """(fewest, most) images one CTA runs: CTA c takes b = c, c + grid, ... (fused_kernels.cu:67, lenet5_kernels.cu:81)"""
    return B // grid, -(-B // grid)


def eval_batches(sm_count):
    """[(B, images the busiest CTA must run)] for the evaluation pass: one image past the cap, seven past twice the cap, the
    fixture, the fixture tiled eight times"""
    cap = fused_grid(sm_count, 1 << 30)
    return [(cap + 1, 2), (2 * cap + 7, 3), (NB, 3), (8 * NB, 3)]


def l5_batches(sm_count):
    """[(B, images the busiest CTA must run)] for the LeNet-5 gradient: one past the cap, one short of twice the cap, the
    fixture; 8 * NB (tiled) runs on its own"""
    cap = l5_grid(sm_count, 1 << 30)
    return [(cap + 1, 2), (2 * cap - 1, 2), (NB, 3)]


# ---------------------------------------------------------------- batched operator tier: grid-stride laps
OPS_MAX_BLOCKS = 148 * 32       # ops_kernels.cu:31


def blocks_for(n, threads):
    """ops_kernels.cu:28-33"""
    b = (n + threads - 1) // threads
    if b < 1:
        b = 1
    if b > OPS_MAX_BLOCKS:
        b = OPS_MAX_BLOCKS
    return b


# op -> (grid-stride items per sample, threads per block, launch line of ops_kernels.cu, text of that line)
OPS = {
    "fp_c1": (3456, 256, 316, "k_fp_c1<<<blocks_for((long)B * PCNN_C1, 256), 256, 0, ctx->stream>>>"),
    "bp_output_c1": (3456, 256, 386, "k_bp_output_c1<<<blocks_for((long)B * PCNN_C1, 256), 256, 0, ctx->stream>>>"),
    "bp_preact_c1": (3456, 256, 392, "k_bp_preact_c1<<<blocks_for((long)B * PCNN_C1, 256), 256, 0, ctx->stream>>>(dpre, dout, pre, (long)B * PCNN_C1);"),
    "apply_step_function": (3456, 256, 283, "k_apply_step<<<blocks_for(n, 256), 256, 0, ctx->stream>>>(in, out, n);"),   # n = B * 3456 here
    "bp_weight_c1": (150, 64, 401, "k_bp_weight_c1_partial<<<blocks_for((long)B * 150, 64), 64, 0, ctx->stream>>>"),
    "fp_s1": (216, 128, 322, "k_fp_s1<<<blocks_for((long)B * PCNN_S1, 128), 128, 0, ctx->stream>>>"),
    "bp_output_s1": (216, 128, 352, "k_bp_output_s1<<<blocks_for((long)B * PCNN_S1, 128), 128, 0, ctx->stream>>>"),
    "bp_preact_s1": (216, 128, 358, "k_bp_preact_s1<<<blocks_for((long)B * PCNN_S1, 128), 128, 0, ctx->stream>>>(dpre, dout, pre, (long)B * PCNN_S1);"),
    "bp_weight_s1": (16, 64, 367, "k_bp_weight_s1_partial<<<blocks_for((long)B * 16, 64), 64, 0, ctx->stream>>>"),
    "fp_preact_f": (10, 64, 328, "k_fp_preact_f<<<blocks_for((long)B * PCNN_F, 64), 64, 0, ctx->stream>>>"),
    "bp_bias_c1": (6, 64, 412, "k_sum576_partial<<<blocks_for((long)B * 6, 64), 64, 0, ctx->stream>>>"),
    "fp_bias_f": (10, 128, 334, "k_fp_bias_f<<<blocks_for((long)B * PCNN_F, 128), 128, 0, ctx->stream>>>"),
    "makeError_batch": (10, 256, 295, "k_make_error<<<blocks_for((long)B * PCNN_F, 256), 256, 0, ctx->stream>>>"),
    "bp_bias_s1": (1, 64, 378, "k_sum216_partial<<<blocks_for(B, 64), 64, 0, ctx->stream>>>"),
    "vectorNorm": (1, 128, 310, "k_vector_norm<<<blocks_for(B, 128), 128, 0, ctx->stream>>>"),
}
SOURCE += [("ops_kernels.cu", line, text) for _, _, line, text in OPS.values()]


def ops_laps(op, B):
    """(blocks, threads, laps) of `op` at batch B: the grid-stride loop of its busiest thread runs `laps` times"""
    per, threads = OPS[op][:2]
    items = B * per
    blocks = blocks_for(items, threads)
    return blocks, threads, -(-items // (blocks * threads))


def ops_min_batch(op):
    """the smallest B at which `op` takes a second lap: B * items > OPS_MAX_BLOCKS * threads"""
    per, threads = OPS[op][:2]
    return OPS_MAX_BLOCKS * threads // per + 1


def ops_batch(op):
    """NB past the first B with a second lap: every fixture digit is in the batch, and the second lap holds NB samples or more"""
    return ops_min_batch(op) + NB


# ---------------------------------------------------------------- planar extension ops
def grid_for(sm_count, items, threads):
    """ext_kernels.cu:11-16"""
    b = (items + threads - 1) // threads
    cap = sm_count * 8
    if b > cap:
        b = cap
    return b if b >= 1 else 1


def maxpool_laps(sm_count, planes, H, W, k):
    """((grid, laps) forward, (grid, laps) backward): one thread per output forward (:107-108), per input backward (:120-121)"""
    out = []
    for total in (planes * (H // k) * (W // k), planes * H * W):
        g = grid_for(sm_count, total, 256)
        out.append((g, -(-total // (g * 256))))
    return tuple(out)


def softmax_laps(sm_count, B):
    """(grid, rows per lap, laps): one warp per row (:131, :81)"""
    g = grid_for(sm_count, B * 32, 256)
    rows = g * 256 // 32
    return g, rows, -(-B // rows)


MAXPOOL_CASES = [(6 * 1024, 24, 24, 2), (6 * 2048, 24, 24, 4)]     # k = 4 is the float4 path
SOFTMAX_CASES = [(20000, 10), (9000, 37)]
