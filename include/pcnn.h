/*
 * include/pcnn.h -- C ABI of the H100-native LeNet/MNIST training engine (libpcnn.so).
 *
 * This is the drop-in boundary for the hot path of Tamerkobba/Parallel-CNN: the 18 layer functions of
 * Sequential/layer.h and the driver entry points of Sequential/Main.cpp.  The reference has no FFI layer
 * (its boundary is `#include "layer.h"`), so include/layer.h in this repo re-declares the reference's own
 * class and functions and forwards each of them to the entry points below; INTEGRATION.md shows the binding.
 * Every entry point cites the reference interface it replaces as  [ref: <file>:<lines>]  relative to
 * /root/reference/.
 *
 * Conventions
 *   - plain C: pointers, sizes, ints.  No torch / C++ types.  All functions return 0 on success or a negative
 *     pcnn_status; pcnn_last_error_string() describes the most recent failure on the calling thread.
 *   - "dev" pointers are CUDA device pointers on the context's device; "host" pointers are ordinary memory.
 *   - every call enqueues on the context's stream; only *_sync / *_d2h / get_* / *_host calls block.
 *   - one context per GPU, not thread-safe per context (the reference is single-threaded global state).
 *   - there is NO CPU fallback: on a machine without a usable sm_90 GPU pcnn_create fails with
 *     PCNN_ERR_NOGPU and nothing else computes.
 *
 * Packed parameter vector (PCNN_NPARAM = 2,343 floats), also the layout of the packed gradient:
 *     [0,150) c1.weight[6][5][5] | [150,156) c1.bias | [156,172) s1.weight[1][4][4] | [172] s1.bias |
 *     [173,2333) f.weight[10][6][6][6] | [2333,2343) f.bias             [ref: Sequential/Main.cpp:17-20]
 * The packed gradient holds what the reference multiplies by dt (the NEGATIVE gradient, layer.h:93): d_weight
 * for the weight blocks and the raw bias accumulators (sum d_preact) for the bias blocks; the /576 and /216
 * of layer.h:412 and layer.h:316 are applied by the update.  Element PCNN_NPARAM of the device-side vector
 * carries the sum of per-sample error norms (Main.cpp:168-169).
 */
#ifndef PCNN_H_
#define PCNN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PCNN_NPARAM 2343
#define PCNN_OFF_C1W 0
#define PCNN_OFF_C1B 150
#define PCNN_OFF_S1W 156
#define PCNN_OFF_S1B 172
#define PCNN_OFF_FW 173
#define PCNN_OFF_FB 2333
#define PCNN_IMG 784   /* 28 x 28 */
#define PCNN_C1 3456   /* 6 x 24 x 24 */
#define PCNN_S1 216    /* 6 x 6 x 6 */
#define PCNN_F 10

typedef enum {
    PCNN_OK = 0,
    PCNN_ERR_ARG = -1,    /* null pointer, negative size, bad enum */
    PCNN_ERR_CUDA = -2,   /* a CUDA runtime call or kernel failed */
    PCNN_ERR_NCCL = -3,   /* NCCL missing or a collective failed */
    PCNN_ERR_STATE = -4,  /* call not valid in the current state (no dataset bound, comm not initialised...) */
    PCNN_ERR_IO = -5,     /* file problems other than the mnist_load codes */
    PCNN_ERR_NOGPU = -6   /* no CUDA device / not compute capability 9.0 */
} pcnn_status;

#define PCNN_MAX_PEERS 8   /* GPUs of one NVSwitch domain the in-kernel gradient exchange addresses */
typedef enum { PCNN_MODE_AUTO = 0, PCNN_MODE_GRAPH = 1, PCNN_MODE_PERSISTENT = 2 } pcnn_step_mode;
typedef enum { PCNN_U8 = 0, PCNN_F32 = 1 } pcnn_pixel_type;   /* IDX bytes, or the reference's float[28][28] */
typedef enum { PCNN_TRAIN_SET = 0, PCNN_TEST_SET = 1 } pcnn_split;

typedef struct pcnn_ctx pcnn_ctx;

/* ------------------------------------------------------------------ library / context */
int pcnn_version(void);
const char *pcnn_last_error_string(void);
/* device < 0: current device.  stream: a cudaStream_t to enqueue on (e.g. the caller's torch stream) or NULL
 * for a private non-blocking stream. */
int pcnn_create(pcnn_ctx **out, int device, void *stream);
int pcnn_destroy(pcnn_ctx *ctx);
int pcnn_sync(pcnn_ctx *ctx);
int pcnn_device_info(pcnn_ctx *ctx, int *sm_count, int *cc_major, int *cc_minor, size_t *hbm_bytes);

/* ------------------------------------------------------------------ device buffers owned by `Layer`
 * [ref: Sequential/layer.h:39-79  Layer::Layer / ~Layer / setOutput / clear / bp_clear] */
int pcnn_malloc(pcnn_ctx *ctx, void **dev, size_t bytes);             /* zero-initialised, like new float[n]() */
int pcnn_free(pcnn_ctx *ctx, void *dev);
int pcnn_memset0(pcnn_ctx *ctx, void *dev, size_t bytes);            /* Layer::clear, Layer::bp_clear */
int pcnn_h2d(pcnn_ctx *ctx, void *dev, const void *host, size_t bytes);   /* Layer::setOutput (blocking) */
int pcnn_d2h(pcnn_ctx *ctx, void *host, const void *dev, size_t bytes);   /* host reads of l_f.output etc. */
int pcnn_d2d(pcnn_ctx *ctx, void *dst, const void *src, size_t bytes);

/* ------------------------------------------------------------------ parameters
 * pcnn_init_params_reference replays the constructor draws of the three static Layer objects: glibc rand()
 * with the default seed, per neuron bias then weights, c1 -> s1 -> f  [ref: layer.h:48-54, Main.cpp:17-20].
 * It is a host-side utility (private re-implementation of the glibc TYPE_3 generator; global rand() state
 * is not touched) and needs no GPU. */
int pcnn_init_params_reference(float *host_params);
int pcnn_set_params(pcnn_ctx *ctx, const float *host_params);
int pcnn_get_params(pcnn_ctx *ctx, float *host_params);
int pcnn_get_grads(pcnn_ctx *ctx, float *host_grads);                /* packed gradient of the last step */
int pcnn_params_dev(pcnn_ctx *ctx, float **dev_params);              /* the context's own packed vector */
int pcnn_set_learning_rate(pcnn_ctx *ctx, float dt);                 /* default 0.1f  [ref: layer.h:12] */
/* 9,372-byte packed checkpoint with a 16-byte header (the reference has none; SURVEY.md 8f.3) */
int pcnn_save_params(pcnn_ctx *ctx, const char *path);
int pcnn_load_params(pcnn_ctx *ctx, const char *path);

/* ------------------------------------------------------------------ per-operator API (drop-in for layer.h)
 * Device pointers; row-major arrays shaped as in the reference with a leading batch dimension B (B = 1 is the
 * reference call).  Arithmetic follows the reference's evaluation order in fp32 without FMA contraction and
 * evaluates the sigmoid in double, so B = 1 results are bit-identical to Sequential/layer.h up to the last-ulp
 * difference between CUDA's and glibc's double exp().  For B > 1 the weight-gradient ops sum over the batch
 * and the in-place bias updates use dt / B (DESIGN.md "mini-batch semantics"). */
int pcnn_apply_step_function(pcnn_ctx *ctx, const float *in, float *out, long n);        /* [ref: layer.h:85-89] */
int pcnn_make_error(pcnn_ctx *ctx, float *err, const float *out, unsigned Y, int n);     /* [ref: layer.h:91-95] */
int pcnn_make_error_batch(pcnn_ctx *ctx, float *err, const float *out, const uint8_t *labels, int B);
int pcnn_apply_grad(pcnn_ctx *ctx, float *w, const float *g, long n);                    /* [ref: layer.h:97-101] */
int pcnn_apply_grad_scaled(pcnn_ctx *ctx, float *w, const float *g, long n, float step);
int pcnn_vector_norm(pcnn_ctx *ctx, const float *v, int n, int B, float *norms_dev);     /* [ref: Main.cpp:28-34] */
int pcnn_fp_c1(pcnn_ctx *ctx, const float *in, float *pre, const float *w, const float *b, int B);   /* [ref: layer.h:105-140] */
int pcnn_fp_s1(pcnn_ctx *ctx, const float *in, float *pre, const float *w, const float *b, int B);   /* [ref: layer.h:143-181] */
int pcnn_fp_preact_f(pcnn_ctx *ctx, const float *in, float *pre, const float *w, int B);             /* [ref: layer.h:184-203] */
int pcnn_fp_bias_f(pcnn_ctx *ctx, float *pre, const float *b, int B);                                /* [ref: layer.h:206-211] */
int pcnn_bp_weight_f(pcnn_ctx *ctx, float *dw, const float *dpre, const float *pout, int B);         /* [ref: layer.h:214-227] */
int pcnn_bp_bias_f(pcnn_ctx *ctx, float *bias, const float *dpre, int B);                            /* [ref: layer.h:229-234] */
int pcnn_bp_output_s1(pcnn_ctx *ctx, float *dout, const float *nw, const float *ndpre, int B);       /* [ref: layer.h:237-257] */
int pcnn_bp_preact_s1(pcnn_ctx *ctx, float *dpre, const float *dout, const float *pre, int B);       /* [ref: layer.h:260-270] */
int pcnn_bp_weight_s1(pcnn_ctx *ctx, float *dw, const float *dpre, const float *pout, int B);        /* [ref: layer.h:272-300] */
int pcnn_bp_bias_s1(pcnn_ctx *ctx, float *bias, const float *dpre, int B);                           /* [ref: layer.h:302-317] */
int pcnn_bp_output_c1(pcnn_ctx *ctx, float *dout, const float *nw, const float *ndpre, int B);       /* [ref: layer.h:319-346] */
int pcnn_bp_preact_c1(pcnn_ctx *ctx, float *dpre, const float *dout, const float *pre, int B);       /* [ref: layer.h:348-369] */
int pcnn_bp_weight_c1(pcnn_ctx *ctx, float *dw, const float *dpre, const float *pout, int B);        /* [ref: layer.h:371-395] */
int pcnn_bp_bias_c1(pcnn_ctx *ctx, float *bias, const float *dpre, int B);                           /* [ref: layer.h:398-414] */

/* ------------------------------------------------------------------ data  [ref: Sequential/mnist.h:79-160, Main.cpp:36-42]
 * pcnn_mnist_load_u8 keeps mnist_load's return codes (0 ok, -1 no such files, -2 bad image file, -3 bad label
 * file, -4 count mismatch) but returns the raw u8 pixels instead of the double[28][28] staging. */
int pcnn_mnist_load_u8(const char *image_file, const char *label_file, uint8_t **images, uint8_t **labels,
                       unsigned *count);
void pcnn_mnist_free(void *p);
/* copy a host dataset to the device and bind it as the train / test split (u8 IDX payload or float[784]) */
int pcnn_dataset_upload(pcnn_ctx *ctx, int split, const void *host_images, int pixel_type,
                        const uint8_t *host_labels, long n);
/* bind caller-owned device buffers instead (no copy; caller keeps them alive) */
int pcnn_dataset_bind(pcnn_ctx *ctx, int split, const void *dev_images, int pixel_type,
                      const uint8_t *dev_labels, long n);

/* ------------------------------------------------------------------ fused training / evaluation path
 * One step = forward_pass + makeError + vectorNorm + back_pass for every sample of the batch with frozen
 * parameters, batch-sum of the packed gradient, (optional all-reduce), update  w += (dt / B_global) * g.
 * At B = 1 this is the body of learn()'s loop  [ref: Main.cpp:157-171, 59-144]. */
int pcnn_train_step(pcnn_ctx *ctx, long first, int B);                 /* samples [first, first+B) of the bound train split */
/* consecutive batches starting at `first` (or continuing at the device-side cursor when first == -1), wrapping at the
 * end of the split; replayed from cached CUDA graphs.  _prepare instantiates the graphs such a call needs (untimed). */
int pcnn_train_steps(pcnn_ctx *ctx, long first, int B, int nsteps);
int pcnn_train_steps_prepare(pcnn_ctx *ctx, int B, int nsteps);
int pcnn_train_step_dev(pcnn_ctx *ctx, const void *dev_images, int pixel_type, const uint8_t *dev_labels, int B);
/* host buffers in, H2D inside the call, error-norm sum of the step back out (blocking) */
int pcnn_train_step_host(pcnn_ctx *ctx, const void *host_images, int pixel_type, const uint8_t *host_labels,
                         int B, float *err_sum_out);
/* frozen-parameter gradient only (no update): fills the packed gradient (+ error sum); used by parity tests */
int pcnn_compute_grads(pcnn_ctx *ctx, const void *dev_images, int pixel_type, const uint8_t *dev_labels, int B);
/* learn(): `epochs` passes over the bound train split in dataset order with batch B (tail batch kept);
 * mean_err_out = sum of error norms / n of the LAST epoch, as learn() prints  [ref: Main.cpp:146-184] */
int pcnn_learn(pcnn_ctx *ctx, int B, int epochs, float *mean_err_out);
/* same, with the dataset in HOST memory.  Page-locked images (cudaHostAlloc / cudaHostRegister, 16-byte aligned): the training
 * kernel reads them across PCIe itself, one image per CTA and step, a step ahead -- no staging copy, one label copy + one launch
 * per epoch.  Pageable images: staged through a chunked H2D copy stream that the kernel follows chunk by chunk.  Same samples,
 * same order, bit-identical results either way; returns when the last step's results are in host memory. */
int pcnn_learn_host(pcnn_ctx *ctx, const void *host_images, int pixel_type, const uint8_t *host_labels,
                    long n, int B, int epochs, float *mean_err_out);
int pcnn_err_sum(pcnn_ctx *ctx, double *sum_out, int reset);           /* running sum of per-sample error norms */
/* forward_pass for B samples; f_out_dev [B][10] may be NULL, pred_dev [B] (first-max argmax) may be NULL
 * [ref: Main.cpp:59-105, 186-200] */
int pcnn_forward_batch(pcnn_ctx *ctx, const void *dev_images, int pixel_type, int B, float *f_out_dev,
                       uint8_t *pred_dev);
/* test(): misclassification count over the bound test split  [ref: Main.cpp:202-214] */
int pcnn_test(pcnn_ctx *ctx, long *wrong_out);
/* number of kernels this context has launched since creation (bench.py's gpu_launches) */
int pcnn_launch_count(pcnn_ctx *ctx, long *count_out);
/* per-step error sums recorded by the most recent pcnn_learn_host epoch (device -> pinned host, one float per step) */
int pcnn_step_errs(pcnn_ctx *ctx, float *host_out, long cap, long *count_out);
/* measurement helpers for bench.py (CUDA events on the context's stream, after `iters / 10 + 3` warm-up launches):
 * average duration of the fused gradient kernel alone over `iters` launches walking the bound train split, and the
 * sustained fp32 FMA rate of this GPU under its current clocks (dependent-chain-free FFMA micro-benchmark). */
int pcnn_time_fused_kernel(pcnn_ctx *ctx, int B, int iters, float *avg_ms_out);
int pcnn_measure_fp32_peak(pcnn_ctx *ctx, float *tflops_out);
/* streaming-read rate (GB/s) of a TMA load pipeline with no consumer work over a bf16 tensor [N][P][Q][64] in HBM:
 * mode 0 = 1-D bulk copies of 16 KB, 1 = 2-D boxes of 128 pixels, 2 = the input-gradient kernel's pattern (boxes of
 * 1 pixel x 32 rows), 3 = the weight-gradient kernel's pattern (one row of pixels per box).  The ceiling the convolution
 * backward kernels are measured against next to the HBM copy peak. */
int pcnn_measure_tma_read(pcnn_ctx *ctx, const void *dev_bf16, int N, int P, int Q, int mode, int iters, float *gbps_out);
/* store rate (GB/s) of the forward convolution's epilogue with everything but the stores removed: y viewed as [N][P][row_elems]
 * bf16, tiles of 128 rows x 256 columns walked like the forward kernel (image height H on the input side, H % 32 == 0).  mode 0 =
 * boxes {64 columns, 32 rows} with 128-byte swizzle, 1 / 2 = boxes of 128 / 256 columns without swizzle,
 * 3 = per-row 1-D bulk stores of 128 bytes, 4 = four boxes per commit group, 5 = 16-byte st.global.v4 from registers (no TMA),
 * 6 = half TMA boxes, half direct stores; hot = 1 aims every tile at the first row block (an
 * L2-resident target).  The ceiling the forward kernel's store phase is measured against.  The tensor is OVERWRITTEN with
 * unspecified values (the staging buffers are never filled). */
int pcnn_measure_tma_write(pcnn_ctx *ctx, void *dev_bf16, int N, int P, int H, int row_elems, int mode, int hot, int iters, float *gbps_out);
/* SM clocks per M x N x 16 bf16 product on the wgmma tensor cores (operands K- or MN-major in shared memory) when each of the
 * M / 64 warpgroups issues `reps` m64nNk16 back to back into one register accumulator: the issue-rate table the convolution
 * kernels are designed against (small-N instructions are far from the tensor-pipe peak).  `nacc` (1, 2, 4, 8 with
 * N * nacc <= 512) is validated only: register accumulators are not rotated. */
int pcnn_measure_mma_rate(pcnn_ctx *ctx, int M, int N, int a_mn_major, int b_mn_major, int nacc, int reps, float *clk_per_mma);

/* ------------------------------------------------------------------ data parallelism (not in the reference; SURVEY.md 8e)
 * Sample-sharded replicas, one process per GPU.  After pcnn_comm_init_rank every train step all-reduces the
 * packed gradient (2,344 floats) once and divides the step by B * world. */
int pcnn_comm_unique_id(void *id_out, size_t *id_bytes);               /* rank 0; 128 bytes */
int pcnn_comm_init_rank(pcnn_ctx *ctx, const void *id, int rank, int world);
int pcnn_comm_destroy(pcnn_ctx *ctx);
int pcnn_allreduce_grads(pcnn_ctx *ctx);
/* In-kernel exchange over NVLink / NVSwitch peer memory (no NCCL launch per step): every rank exports one IPC handle
 * (64 bytes) for its inbox, the handles of all ranks are gathered by any rendezvous and attached.  Afterwards the
 * persistent training kernel pushes its chunk of the reduced gradient straight into every peer's inbox and adds the
 * ranks' chunks in rank order, inside the step. */
int pcnn_p2p_export(pcnn_ctx *ctx, void *handle_out, size_t *handle_bytes);
int pcnn_p2p_attach(pcnn_ctx *ctx, const void *handles, int rank, int world);
int pcnn_p2p_detach(pcnn_ctx *ctx);
/* How cursor-driven steps (pcnn_train_steps, pcnn_learn, pcnn_learn_host) execute: PCNN_MODE_PERSISTENT = one
 * cooperative kernel running all steps (thread-block clusters + tagged words through L2 instead of grid barriers,
 * in-kernel reduction/update/exchange); PCNN_MODE_GRAPH = CUDA graphs of per-step kernels (+ NCCL all-reduce when
 * distributed); PCNN_MODE_AUTO (default) = persistent whenever it can serve the configuration (single GPU, or peers
 * attached), else graph. */
int pcnn_set_step_mode(pcnn_ctx *ctx, int mode);
/* Geometry of the most recent persistent launch and what the device can hold: out6 = { grid, cluster size, co-resident CTAs,
 * co-resident CTAs when launched as clusters, the cluster size the kernel is built for, 1 if the launches are cooperative }.
 * pcnn_persist_tune(ctx, mask): bit 0 forces the variant without clusters; bit 1 keeps the clusters but launches without the
 * cooperative attribute (profilers that re-issue cooperative launches drop the cluster dimension); bit 2 makes
 * pcnn_learn_host enqueue its host copies BEFORE the kernel launch (needed wherever launches block the calling thread:
 * kernel-replay profilers; CUDA_LAUNCH_BLOCKING=1 is detected by itself); bit 3 keeps the two-stage gradient exchange on 2
 * GPUs (default there: cluster shares stored straight into the peer's memory); bit 4 sends pinned host images of
 * pcnn_learn_host through the staged copy stream instead of letting the kernel pull them.  Measurement knobs for A/B runs.
 * Each call sets every knob from its mask, so pcnn_persist_tune(ctx, 0) restores the defaults; a driver that refused a
 * cooperative cluster launch and CUDA_LAUNCH_BLOCKING=1 still keep bits 1 and 2 on, as they do without any tune call.
 * out6[5] of pcnn_persist_info: bit 0 = cooperative launch, bit 1 = direct exchange used, bit 2 = two images per CTA (one
 * 448-thread CTA per SM, chosen when the batch outnumbers the SMs and ceil(B / 2) such CTAs fit as clusters). */
int pcnn_persist_info(pcnn_ctx *ctx, int *out6);
int pcnn_persist_tune(pcnn_ctx *ctx, int max_cluster);
/* Phase timestamps of the persistent kernel (ns; 6 per step: step start, parameters resident, images done, cluster slot
 * written, owned chunk gathered, parameters published; first 256 steps of a launch, CTA 0).  host_out == NULL arms tracing for the
 * following launches, host_out != NULL reads the stamps back. */
int pcnn_persist_trace(pcnn_ctx *ctx, long long *host_out, int cap_steps);
/* the same six stamps of EVERY CTA at step 128 of the traced launch, rows of 8 (six stamps, SM id, spare): their spread is
 * the skew between CTAs that the gradient owners have to wait for */
int pcnn_persist_trace_ctas(pcnn_ctx *ctx, long long *host_out, int cap_ctas);

/* ------------------------------------------------------------------ north_star extension ops (parity unpinned by the reference)
 * max-pool k x k stride k over [C][H][W] planes with argmax cache (flat index i*k+j, first maximum wins) */
int pcnn_maxpool_fwd(pcnn_ctx *ctx, const float *in, float *out, int32_t *argmax, int planes, int H, int W, int k);
int pcnn_maxpool_bwd(pcnn_ctx *ctx, const float *dout, const int32_t *argmax, float *din, int planes, int H, int W, int k);
/* softmax cross-entropy over n logits per row; d = onehot - p (the reference's sign convention for d_preact) */
int pcnn_softmax_ce(pcnn_ctx *ctx, const float *logits, const uint8_t *labels, int B, int n, float *prob,
                    float *d, float *loss);

/* ------------------------------------------------------------------ LeNet-5-style variant with a second convolution layer
 * (SURVEY.md 8f row 4; PARITY UNPINNED: the reference has exactly one conv layer, layer.h:105-140 / Main.cpp:17-20).
 *     28x28 -> c1 6@5x5 -> s2 shared 2x2/2 weighted sum -> c3 16@5x5 over 6 channels -> s4 shared 2x2/2 -> f 256 -> 10,
 * sigmoid everywhere, the reference's loss (d_preact_f = onehot - output) and its gradient / update rules generalised by
 * rule; oracle/lenet5_oracle.c is the definition.  Packed parameters, PCNN_L5_NPARAM = 5,152 floats:
 *     c1w 150 | c1b 6 | s2w 4 | s2b 1 | c3w [16][6][5][5] 2400 | c3b 16 | s4w 4 | s4b 1 | fw [10][256] 2560 | fb 10.
 * All pointers are device pointers; grads_dev holds PCNN_L5_NPARAM + 1 floats (packed gradient, then the batch sum of
 * error norms) and may be NULL for pcnn_l5_train_step.  One fused kernel per batch (activations and parameters in shared
 * memory) + a fixed-order slot reduction: deterministic.  Update: w += (dt / B) * g with the bias divisors of the rules. */
#define PCNN_L5_NPARAM 5152
int pcnn_l5_compute_grads(pcnn_ctx *ctx, const float *params_dev, const void *images_dev, int pixel_type,
                          const uint8_t *labels_dev, int B, float *grads_dev);
int pcnn_l5_train_step(pcnn_ctx *ctx, float *params_dev, const void *images_dev, int pixel_type, const uint8_t *labels_dev,
                       int B, float *grads_dev);
int pcnn_l5_forward(pcnn_ctx *ctx, const float *params_dev, const void *images_dev, int pixel_type, int B, float *f_out_dev);

/* ------------------------------------------------------------------ bf16 tensor-core convolution (SURVEY.md x3; BASELINE configs 3, 5)
 * The reference's conv semantics (valid, stride 1, cross-correlation, layer.h:118-130) generalised to C input channels,
 * K filters of R x S taps, on the wgmma tensor cores with register accumulators and TMA-fed operands (csrc/conv_tc.cu).
 * Activations are NHWC bf16 with a row pitch of `row_pitch` elements (>= W*C, multiple of 8); filters fp32 KRSC on the
 * host (rounded to bf16 on the device at plan creation, refreshed from device memory by pcnn_conv_plan_set_params); output NHWC bf16 [N][H-R+1][W-S+1][K], bias and activation
 * (act 0 none, 1 sigmoid, 3 ReLU: PCNN_ACT_* below) fused.
 * Pad contents are ignored by the forward, the weight gradient and the input gradient alike: the pad columns W*C ..
 * row_pitch-1 and the pad rows H .. image_rows-1 of x may hold anything, NaN included, without changing a result bit.
 * Constraint of this round: some pixel block Qt with (Qt+S-1)*C <= 32, Qt*K <= 256 and Qt*K % 16 == 0 must exist
 * (LeNet c1: Qt = 24; 224x224x3 -> 64 x 3x3: Qt = 4).  PARITY UNPINNED by the reference (it has no bf16 path): the
 * checker is orc_conv_fwd_nhwc in oracle/lenet_oracle.c on the bf16-rounded operands. */
/* Activation codes (`act`) of the device-trained layers: every create call below (row-Toeplitz, wide, padded wide, linear) and
 * pcnn_conv_bias_act_bwd take one of these three; any other value, 2 included, is PCNN_ERR_ARG with the message
 * "<function>: act <n> is not 0 (none), 1 (sigmoid) or 3 (ReLU)".  The forward epilogue first forms v = fp32 accumulator + bias,
 * then
 *   PCNN_ACT_NONE:    y = bf16_rn(v);
 *   PCNN_ACT_SIGMOID: y = bf16_rn(sigmoid(v)) (the reference's activation, layer.h:81-83);
 *   PCNN_ACT_RELU:    y = bf16_rn(v < 0 ? +0 : v), applied once in fp32 before the one rounding.  NaN and -0 pass unchanged, as
 *                     in torch.relu / clamp_min(0) (not fmaxf, which turns NaN into 0): +Inf stays +Inf, -Inf gives +0, a
 *                     negative v gives +0 and a positive v too small for bf16 rounds to +0.
 * The backward of each is pcnn_conv_bias_act_bwd with the same code. */
#define PCNN_ACT_NONE 0
#define PCNN_ACT_SIGMOID 1
#define PCNN_ACT_RELU 3
/* Codes 4-6 are taken by pcnn_batchnorm_nhwc_bf16_fwd and pcnn_batchnorm_nhwc_bf16_bwd_preact, and by group normalization's
 * forward and pre-activation backward, only (every other call above and below keeps its domain and refuses them); batch
 * normalization below states their formulas. */
#define PCNN_ACT_SILU 4
#define PCNN_ACT_HARDSWISH 5
#define PCNN_ACT_RELU6 6
typedef struct pcnn_conv_plan pcnn_conv_plan;
int pcnn_conv_tc_plan_create(pcnn_ctx *ctx, int N, int H, int W, int C, int K, int R, int S, int row_pitch,
                             int image_rows /* rows between consecutive images in memory, >= H; 0 = H */,
                             int act, const float *filt_host, const float *bias_host, pcnn_conv_plan **plan_out);
/* the same with a window step of `stride` (1..4) in both directions (SURVEY.md 8f row 4): y [N][(H-R)/stride+1][(W-S)/stride+1][K];
 * rows per image (image_rows, or H) must be a multiple of the stride; the pixel block then needs ((Qt-1)*stride+S)*C <= 32.
 * Its backward passes are pcnn_conv_wgrad_strided / pcnn_conv_dgrad_strided. */
int pcnn_conv_tc_plan_create_strided(pcnn_ctx *ctx, int N, int H, int W, int C, int K, int R, int S, int stride, int row_pitch,
                                     int image_rows, int act, const float *filt_host, const float *bias_host,
                                     pcnn_conv_plan **plan_out);
int pcnn_conv_tc_plan_destroy(pcnn_ctx *ctx, pcnn_conv_plan *plan);
/* Host-only query (works without a GPU and without a context): how pcnn_conv_tc_plan_create_strided tiles a shape.
 * out5 = { Qt output pixels per tile, V Toeplitz alignment variants, activation stages, row tiles of 128 rows, pixel tiles per row }.
 * The persistent kernel runs min(tiles, SMs) CTAs over the n_mtiles * n_qtiles tiles.  Shapes the plan refuses return the same
 * error here. */
int pcnn_conv_tc_plan_info(int N, int H, int W, int C, int K, int R, int S, int stride, int row_pitch, int image_rows, int *out5);
int pcnn_conv_tc_fwd(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *x_bf16_dev, void *y_bf16_dev);
/* Forward for wide channel counts (csrc/conv_wide_tc.cu): the same contract as pcnn_conv_tc_plan_create_strided (x NHWC bf16 with
 * row_pitch and image_rows, filters fp32 KRSC rounded to bf16 here or by pcnn_conv_plan_set_params, optional bias, act 0 none / 1 sigmoid / 3 ReLU, y dense NHWC bf16
 * [N][(H-R)/stride+1][(W-S)/stride+1][K], pad columns and pad rows of x ignored, NaN included), computed as a tap-major implicit
 * GEMM on wgmma with the channels as the reduction.  The plan is run by pcnn_conv_tc_fwd (which then also needs y 16-byte aligned)
 * and freed by pcnn_conv_tc_plan_destroy.  Its domain is exactly the shapes that
 *   - pcnn_conv_tc_plan_info refuses (a shape the row-Toeplitz plan takes is refused here with a message naming
 *     pcnn_conv_tc_plan_create: no shape has two forward kernels),
 *   - have C % 8 == 0, K % 8 == 0 and K <= 256, 1 <= R, S <= 7, stride 1..4,
 *   - and satisfy the pitch rules (row_pitch >= W*C and a multiple of 8, image_rows >= H or 0 for H).
 * Everything else is PCNN_ERR_ARG with a message naming the rule.  Rows per image need not be a multiple of the stride. */
int pcnn_conv_wide_plan_create(pcnn_ctx *ctx, int N, int H, int W, int C, int K, int R, int S, int stride, int row_pitch,
                               int image_rows, int act, const float *filt_host, const float *bias_host, pcnn_conv_plan **plan_out);
/* Host-only query (no GPU, no context): how pcnn_conv_wide_plan_create tiles a shape; its refusals are the create call's.
 * out8 = { Pt output rows x Qt output columns of one image per tile (Pt * Qt = 128), 64-channel chunks per tap, stages, tiles
 * (N * blocks per image), pixel blocks down a column of the image, pixel blocks along a row, MMA width (K rounded up to 16) }.
 * The tiles issue tiles * 128 output pixels for the N * P * Q they compute. */
int pcnn_conv_wide_plan_info(int N, int H, int W, int C, int K, int R, int S, int stride, int row_pitch, int image_rows, int *out8);
/* Gradients of pcnn_conv_tc_fwd with a plan from pcnn_conv_wide_plan_create (csrc/conv_wide_bwd_tc.cu), on the tensor cores only
 * (pcnn_conv_bwd_select does not apply).  The formulas, dy [N][(H-R)/stride+1][(W-S)/stride+1][K] dense, dw fp32 KRSC and dx bf16
 * in x's layout are those of pcnn_conv_wgrad_strided / pcnn_conv_dgrad_strided: every element of the H x W x C image of dx is
 * written (rows and columns no window covers get 0), pad columns and pad rows of dx are never written, and the pad contents of x
 * are ignored, NaN included.  x, dy and dx must be 16-byte aligned.  The domain is exactly pcnn_conv_wide_plan_info's, refused
 * with the same rule text naming the called function.  Both are deterministic: reruns are bit-identical. */
int pcnn_conv_wide_wgrad(pcnn_ctx *ctx, const void *x_bf16_dev, const void *dy_bf16_dev, float *dw_f32_dev, int N, int H, int W, int C,
                         int K, int R, int S, int stride, int row_pitch, int image_rows);
int pcnn_conv_wide_dgrad(pcnn_ctx *ctx, const void *dy_bf16_dev, const float *filt_f32_dev, void *dx_bf16_dev, int N, int H, int W,
                         int C, int K, int R, int S, int stride, int row_pitch, int image_rows);
/* Host-only query (no GPU, no context): how those two tile a shape; refusals as theirs, naming pcnn_conv_wide_bwd_info.
 * out10 = { weight gradient: row blocks R*S*ceil(C/64) of 64 GEMM rows (a work unit takes two), pixel ranges, pixel blocks per
 *           range (the fewest; the forward's Pt x Qt blocks), stages, work units (row-block pairs x ranges);
 *           input gradient: Pt, Qt of its pixel block of one phase's grid, channel groups, stages, tiles } */
int pcnn_conv_wide_bwd_info(int N, int H, int W, int C, int K, int R, int S, int stride, int row_pitch, int image_rows, int *out10);
/* The same five with a symmetric zero padding of pad_h rows and pad_w columns, as torch.nn.functional.conv2d(padding=(pad_h, pad_w)):
 * with x~ = x inside the H x W image and 0 outside it,
 *     P = (H + 2 pad_h - R) / stride + 1,   Q = (W + 2 pad_w - S) / stride + 1
 *     y[n][p][q][k]  = b[k] + sum_{r,s,c} x~[n][p*stride + r - pad_h][q*stride + s - pad_w][c] * f[k][r][s][c]   (then act)
 *     dw[k][r][s][c] = sum_{n,p,q} dy[n][p][q][k] * x~[n][p*stride + r - pad_h][q*stride + s - pad_w][c]
 *     dx[n][h][w][c] = sum_{k,r,s} dy[n][(h + pad_h - r)/stride][(w + pad_w - s)/stride][k] * f[k][r][s][c]
 *                      over the (r, s) that divide exactly and give a dy pixel inside P x Q:
 * exactly pcnn_pad_nhwc_bf16 into a zeroed canvas followed by the unpadded pass, with dx cropped from the canvas's gradient, but
 * with no canvas: the kernels read x and dy at shifted box coordinates and TMA zero-fills what lies outside.  dy is dense
 * [N][P][Q][K]; out8 / out10 and every other part of the contract are the unpadded calls' (every element of dx's H x W x C image
 * is written, its pad never; the pad columns and rows of x's layout are not the zero padding and are never read, NaN included;
 * reruns are bit-identical).  The domain is the unpadded one with, in addition,
 *   - 0 <= pad_h <= R - 1 and 0 <= pad_w <= S - 1 ("same" is R/2, "full" is R - 1);
 *   - H + 2 pad_h >= R and W + 2 pad_w >= S in place of H >= R and W >= S;
 *   - H >= stride if pad_h > 0 and W >= stride if pad_w > 0 (every phase of x must have a row / pixel inside the image).
 * At padding (0, 0) each is exactly its unpadded call, refusals included (a shape the row-Toeplitz plan takes is refused).
 * A padded shape is never refused for that: the row-Toeplitz plan has no padding, so no shape has two forward kernels.
 * Refusals name the called function (pcnn_conv_wide_plan_create_padded for both forward calls). */
int pcnn_conv_wide_plan_create_padded(pcnn_ctx *ctx, int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w,
                                      int row_pitch, int image_rows, int act, const float *filt_host, const float *bias_host,
                                      pcnn_conv_plan **plan_out);
int pcnn_conv_wide_plan_info_padded(int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w, int row_pitch,
                                    int image_rows, int *out8);
int pcnn_conv_wide_wgrad_padded(pcnn_ctx *ctx, const void *x_bf16_dev, const void *dy_bf16_dev, float *dw_f32_dev, int N, int H, int W,
                                int C, int K, int R, int S, int stride, int pad_h, int pad_w, int row_pitch, int image_rows);
int pcnn_conv_wide_dgrad_padded(pcnn_ctx *ctx, const void *dy_bf16_dev, const float *filt_f32_dev, void *dx_bf16_dev, int N, int H,
                                int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w, int row_pitch, int image_rows);
int pcnn_conv_wide_bwd_info_padded(int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w, int row_pitch,
                                   int image_rows, int *out10);
/* The same five with a dilation (dil_h, dil_w) after the padding, as torch.nn.functional.conv2d(padding=(pad_h, pad_w),
 * dilation=(dil_h, dil_w)) ("atrous" convolution): tap (r, s) sits r*dil_h rows and s*dil_w columns from the window's corner.
 * With the window's extent E_h = dil_h (R - 1) + 1, E_w = dil_w (S - 1) + 1 and x~ as above,
 *     P = (H + 2 pad_h - E_h) / stride + 1,   Q = (W + 2 pad_w - E_w) / stride + 1
 *     y[n][p][q][k]  = b[k] + sum_{r,s,c} x~[n][p*stride - pad_h + r*dil_h][q*stride - pad_w + s*dil_w][c] * f[k][r][s][c]   (then act)
 *     dw[k][r][s][c] = sum_{n,p,q} dy[n][p][q][k] * x~[n][p*stride - pad_h + r*dil_h][q*stride - pad_w + s*dil_w][c]
 *     dx[n][h][w][c] = sum_{k,r,s} dy[n][(h + pad_h - r*dil_h)/stride][(w + pad_w - s*dil_w)/stride][k] * f[k][r][s][c]
 *                      over the (r, s) that divide exactly and give a dy pixel inside P x Q.
 * The forward and the weight gradient run the padded calls' kernels (only the per-tap phase and offset of x change).  The input
 * gradient runs the padded call's kernel with two more steps in its tap walk: with g = gcd(dil_h, stride), row phase a of dx has
 * no taps unless g divides a + pad_h (its elements are written as 0), and otherwise takes the taps r = rho + (stride/g) i, each
 * reading dy row u - (dil_h/g) i + (a + pad_h - rho dil_h)/stride (columns the same).  Each dx element sums in the order of the
 * padded call: ascending i, then j, then 64-filter chunk.  out8 / out10 and every other part of the contract are the padded calls'.
 * The domain is the padded one with, in place of its padding and size rules,
 *   - 1 <= dil_h, dil_w <= 256;
 *   - 0 <= pad_h <= dil_h (R - 1) and 0 <= pad_w <= dil_w (S - 1);
 *   - H + 2 pad_h >= E_h and W + 2 pad_w >= E_w;
 *   - H >= stride if pad_h > 0 and W >= stride if pad_w > 0: a padded direction may read every phase of x, and each phase map
 *     must have a row / pixel inside the image (unpadded, the phases read are (r dil_h) mod stride < E_h <= H).
 * A shape with a dilation other than (1, 1) is never refused for the row-Toeplitz plan (it has no dilation), so no shape has two
 * forward kernels.  At dilation (1, 1) each is exactly its padded call, refusals and their text included, except that refusals
 * name the called function (pcnn_conv_wide_plan_create_dilated for both forward calls). */
int pcnn_conv_wide_plan_create_dilated(pcnn_ctx *ctx, int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w,
                                       int dil_h, int dil_w, int row_pitch, int image_rows, int act, const float *filt_host,
                                       const float *bias_host, pcnn_conv_plan **plan_out);
int pcnn_conv_wide_plan_info_dilated(int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w, int dil_h,
                                     int dil_w, int row_pitch, int image_rows, int *out8);
int pcnn_conv_wide_wgrad_dilated(pcnn_ctx *ctx, const void *x_bf16_dev, const void *dy_bf16_dev, float *dw_f32_dev, int N, int H, int W,
                                 int C, int K, int R, int S, int stride, int pad_h, int pad_w, int dil_h, int dil_w, int row_pitch,
                                 int image_rows);
int pcnn_conv_wide_dgrad_dilated(pcnn_ctx *ctx, const void *dy_bf16_dev, const float *filt_f32_dev, void *dx_bf16_dev, int N, int H,
                                 int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w, int dil_h, int dil_w, int row_pitch,
                                 int image_rows);
int pcnn_conv_wide_bwd_info_dilated(int N, int H, int W, int C, int K, int R, int S, int stride, int pad_h, int pad_w, int dil_h,
                                    int dil_w, int row_pitch, int image_rows, int *out10);
/* Backward passes of the same convolution (bf16 operands, fp32 accumulation, deterministic; wgmma kernels, see
 * pcnn_conv_bwd_select): weight gradient fp32 KRSC [ref: layer.h:371-395 bp_weight_c1, without its /576] and input gradient
 * bf16 NHWC in x's layout.  row_pitch / image_rows as for the forward plan (0 = dense). */
int pcnn_conv_wgrad(pcnn_ctx *ctx, const void *x_bf16_dev, const void *dy_bf16_dev, float *dw_f32_dev, int N, int H, int W, int C,
                    int K, int R, int S, int row_pitch, int image_rows);
int pcnn_conv_dgrad(pcnn_ctx *ctx, const void *dy_bf16_dev, const float *filt_f32_dev, void *dx_bf16_dev, int N, int H, int W,
                    int C, int K, int R, int S, int row_pitch, int image_rows);
/* The same for a window step of `stride` (1..4; anything else is PCNN_ERR_ARG), the gradients of pcnn_conv_tc_fwd with a plan
 * from pcnn_conv_tc_plan_create_strided.  dy is [N][(H-R)/stride+1][(W-S)/stride+1][K], as that forward writes it;
 *     dw[k][r][s][c] = sum_{n,p,q} dy[n][p][q][k] * x[n][p*stride+r][q*stride+s][c]
 *     dx[n][h][w][c] = sum_{k,r,s} dy[n][(h-r)/stride][(w-s)/stride][k] * f[k][r][s][c]   over the (r, s) that divide exactly.
 * Every element of the H x W image of dx is written: rows and columns no window covers ((H-R) % stride != 0,
 * (W-S) % stride != 0, or the gaps between windows when stride > R or S) get 0; pad columns and rows are never written.  The
 * pad rules above hold unchanged, and rows per image need not be a multiple of the stride.  The tensor-core input gradient
 * exists at strides 1 and 2 for 3x3 taps with C in {1,2,3,4,8}, 5x5 with C in {1,3} and 7x7 with C = 1, and at strides 3
 * and 4 for 3x3 taps with C in {1,2,3}; the weight gradient needs ((RB-1)*stride + R)*S*C <= 64 for some RB >= 1.  Stride 1
 * is exactly pcnn_conv_wgrad / pcnn_conv_dgrad. */
int pcnn_conv_wgrad_strided(pcnn_ctx *ctx, const void *x_bf16_dev, const void *dy_bf16_dev, float *dw_f32_dev, int N, int H, int W,
                            int C, int K, int R, int S, int stride, int row_pitch, int image_rows);
int pcnn_conv_dgrad_strided(pcnn_ctx *ctx, const void *dy_bf16_dev, const float *filt_f32_dev, void *dx_bf16_dev, int N, int H, int W,
                            int C, int K, int R, int S, int stride, int row_pitch, int image_rows);
/* Which kernels pcnn_conv_wgrad / pcnn_conv_dgrad may use.  PCNN_CONV_BWD_TENSOR (default): the wgmma kernels only (any filter
 * count up to 256: counts that are not a multiple of 64 are zero-padded to one in an extra pass over dy) -- a shape they
 * cannot take is an ERROR (PCNN_ERR_ARG naming the restriction), never a silent detour.  PCNN_CONV_BWD_REFERENCE: the
 * deterministic FMA-pipe kernels of csrc/conv_bwd.cu for every shape (any C, K, taps): a second implementation the tests
 * compare the tensor-core kernels against, ~1 % of the HBM roofline at BASELINE config 5 -- an explicit opt-in. */
typedef enum { PCNN_CONV_BWD_TENSOR = 0, PCNN_CONV_BWD_REFERENCE = 1 } pcnn_conv_bwd_path;
int pcnn_conv_bwd_select(pcnn_ctx *ctx, int path);
/* Host-only query (works without a GPU): which kernels pcnn_conv_wgrad / pcnn_conv_dgrad pick for a shape and how they tile it.
 * out9 = { wgrad on tensor cores, dy rows per tile, pixels per tile, stages,
 *          dgrad on tensor cores, column strips, output pixels per lane quarter, partial dx rows each consumer thread keeps
 *          in registers (stride * ((R-1)/stride + 1); R at stride 1), stages } */
int pcnn_conv_bwd_plan_info(int N, int H, int W, int C, int K, int R, int S, int *out9);
/* the same for pcnn_conv_wgrad_strided / pcnn_conv_dgrad_strided (stride 1..4, else PCNN_ERR_ARG) */
int pcnn_conv_bwd_plan_info_strided(int N, int H, int W, int C, int K, int R, int S, int stride, int *out9);
/* Zero padding for the valid-padding kernels above (SURVEY.md 8f row 4): pcnn_pad_nhwc_bf16 embeds dense [N][H][W][C] images into
 * a zeroed canvas [N][dst_image_rows][dst_row_pitch] at row offset pad_h, pixel offset pad_w (0 = the tight canvas
 * [H + 2 pad_h][(W + 2 pad_w) * C]); a "same" convolution is pad -> pcnn_conv_tc_fwd, its input gradient is
 * pcnn_conv_dgrad into a padded canvas -> pcnn_crop_nhwc_bf16, its weight gradient is pcnn_conv_wgrad on the padded x.  The wide
 * family pads without a canvas: pcnn_conv_wide_plan_create_padded / pcnn_conv_wide_wgrad_padded / pcnn_conv_wide_dgrad_padded. */
int pcnn_pad_nhwc_bf16(pcnn_ctx *ctx, const void *src_bf16_dev, void *dst_bf16_dev, int N, int H, int W, int C, int pad_h, int pad_w,
                       int dst_row_pitch, int dst_image_rows);
int pcnn_crop_nhwc_bf16(pcnn_ctx *ctx, const void *src_bf16_dev, void *dst_bf16_dev, int N, int H, int W, int C, int pad_h, int pad_w,
                        int src_row_pitch, int src_image_rows);
/* fp32 [rows][w] -> bf16 [rows][pitch] with zero padding (builds the padded activation rows the TMA descriptor needs) */
int pcnn_f32_to_bf16_rows(pcnn_ctx *ctx, const float *src_dev, void *dst_bf16_dev, long rows, int w, int pitch);
/* ------------------------------------------------------------------ training a convolution layer on the device
 * Refresh the parameters of a plan of any kind (pcnn_conv_tc_plan_create[_strided], pcnn_conv_wide_plan_create[_padded]) from
 * device memory: filt_f32_dev fp32 KRSC [K][R][S][C] as the create calls take them from the host, bias_f32_dev fp32 [K].  Either
 * may be NULL ("unchanged"); both NULL is PCNN_ERR_ARG, and so is a bias for a plan created without one.  Enqueued on the
 * context's stream with no host synchronisation and no allocation: a pcnn_conv_tc_fwd enqueued before it reads the old
 * parameters, one enqueued after it the new ones.  The plan's buffers and tensor maps stay; only their contents change.
 * The filters are rounded to bf16 (round to nearest even) on the device, by the same kernels the create calls use for their host
 * filters (uploaded to a temporary device buffer first): a plan refreshed with f holds the same operand bits as a plan created
 * from f.  A NaN filter stays a NaN; its payload is whatever __float2bfloat16_rn makes of it. */
int pcnn_conv_plan_set_params(pcnn_ctx *ctx, pcnn_conv_plan *plan, const float *filt_f32_dev, const float *bias_f32_dev);
/* The activation derivative and the bias gradient of a convolution or linear layer in one pass over dy.  y, dy and dpre are
 * dense bf16 [pixels][K] (pixels = N * P * Q, the layout both forwards write and the gradients read as dy).
 *   act 1: dpre = bf16_rn(float(dy) * (float(y) * (1 - float(y)))), in exactly this order, fp32 round to nearest with no
 *          contraction: the derivative at the pre-activation whose sigmoid the forward stored.  y and dpre must not be NULL.
 *   act 3: dpre = float(y) <= 0 ? +0 : dy, dy's bits passed through with no arithmetic: the ReLU derivative on the output the
 *          forward stored, as torch's threshold_backward(dy, y, 0) (a NaN y passes dy; y = +-0 gives +0).  y and dpre must
 *          not be NULL.
 *   act 0: dpre must be NULL and y is not read; only db is computed, over dy.
 *   db[k] = sum over the pixels of float(dpre[pixel][k]) (of dy at act 0): the bf16 values the weight and input gradients consume,
 *          accumulated in fp32 in a fixed order (per-CTA partials over pixel ranges that depend only on pixels and K, then a
 *          fixed-order pass over them, no atomics): reruns and every H100 give the same bits.  db may be NULL at act 1 and 3
 *          (no bias).
 * dpre == dy (in place) is allowed; no other overlap is.  Domain: 1 <= K <= 256, pixels >= 1, act 0, 1 or 3 (PCNN_ACT_*), every
 * pointer 16-byte aligned; anything else is PCNN_ERR_ARG with the rule in the message.  Elements past pixels * K are never
 * written. */
int pcnn_conv_bias_act_bwd(pcnn_ctx *ctx, const void *y_bf16_dev, const void *dy_bf16_dev, void *dpre_bf16_dev, float *db_f32_dev,
                           long pixels, int K, int act);
/* Max pooling between convolution layers (csrc/pool_nhwc.cu), as torch.nn.functional.max_pool2d with ceil_mode=False and
 * dilation 1, in the layouts of the layers around it:
 *   - x is dense bf16 [N][H][W][C], exactly what both forwards write as y;
 *   - y and dy are [N][image_rows][row_pitch] with P x Q pixels of C channels per image: the layout a plan reads as x;
 *   - dx is dense [N][H][W][C], exactly what pcnn_conv_bias_act_bwd and the weight gradients read as dy;
 *   - argmax is uint8 dense [N][P][Q][C].
 *     P = (H + 2 pad_h - R) / stride + 1,   Q = (W + 2 pad_w - S) / stride + 1.
 * Forward: the window of output (p, q) starts at (h0, w0) = (p stride - pad_h, q stride - pad_w).  Over its positions inside the
 * image only (padding is never a candidate), r = 0..R-1 then s = 0..S-1, starting from m = -Inf and a = the first in-image
 * position, a position is taken when float(v) > m or v is NaN.  So the first maximum wins a tie (-0 and +0 included), the last
 * NaN in the window wins if there is one, and a window of all -Inf gives its first in-image element.  y[n][p][q][c] is the bits
 * of x at the winner, argmax[n][p][q][c] the byte r S + s (< 49).  argmax may be NULL (inference).
 * Backward: dx[n][h][w][c] sums float(dy[n][p][q][c]) over the windows (p, q) that contain (h, w) and whose argmax points at it,
 * in ascending p, then ascending q, in fp32 starting from the first term, rounded to bf16 once (a sum with a NaN term and two or
 * more terms is a NaN whose payload is the conversion's).  With one term dx is dy's bits; with none it is +0.  Every element of
 * the H x W x C image of dx is written, rows and columns no window covers included; there is no memset pass and no atomics.  When
 * stride >= R and stride >= S no element has more than one term.
 * The pad columns and pad rows of y's layout are never written; those of dy are never read (NaN there changes no bit).
 * Domain (anything else is PCNN_ERR_ARG with the function and the rule in the message):
 *   - N, H, W, C >= 1; 1 <= R, S <= 7; stride 1..7 (larger than the window is allowed: the gaps get zero gradient);
 *   - 0 <= pad_h <= R/2 and 0 <= pad_w <= S/2 (every window then holds an image element); H + 2 pad_h >= R, W + 2 pad_w >= S;
 *   - row_pitch 0 = Q C rounded up to a multiple of 8, otherwise >= Q C and a multiple of 8; image_rows 0 = P, otherwise >= P;
 *   - H W C, P Q C and Q C within the 32-bit index range of one image;
 *   - every pointer 16-byte aligned; x, y and argmax pairwise disjoint; dy and argmax disjoint from dx.
 * Both calls are stream-ordered on the context's stream, allocate nothing, and give the same bits on every run and SM count.
 * pcnn_maxpool_nhwc_info: host only (no GPU, no context), refusals as the two calls.  out5 = { P, Q, row pitch used, channels per
 * thread (8 when C % 8 == 0: 16-byte vectors, else 1), most windows over one input pixel }. */
int pcnn_maxpool_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, void *y_bf16_dev, uint8_t *argmax_dev, int N, int H, int W, int C,
                               int R, int S, int stride, int pad_h, int pad_w, int y_row_pitch, int y_image_rows);
int pcnn_maxpool_nhwc_bf16_bwd(pcnn_ctx *ctx, const void *dy_bf16_dev, const uint8_t *argmax_dev, void *dx_bf16_dev, int N, int H, int W,
                               int C, int R, int S, int stride, int pad_h, int pad_w, int dy_row_pitch, int dy_image_rows);
int pcnn_maxpool_nhwc_info(int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int row_pitch, int image_rows,
                           int *out5);
/* Average pooling between convolution layers (csrc/pool_nhwc.cu), in the max pool's layouts, shapes and domain (the refusals read
 * the same, with the function's name), as torch.nn.functional.avg_pool2d with ceil_mode=False and no divisor_override.  Every fp32
 * operation below rounds to nearest with no contraction; "/" is an IEEE division, not a product with a reciprocal.
 *   - count_include_pad must be 0 or 1.  cnt(p, q) = R S when it is 1, else the number of the window's in-image positions (>= 1:
 *     with pad <= R/2 every window holds an image element).  With no ceil mode R S is also torch's divisor.
 * Forward: s = the sum of float(x) over the in-image positions of the window of (p, q), r = 0..R-1 then s = 0..S-1, starting from
 *   the first term (not from +0); y[n][p][q][c] = bf16_rn(s / float(cnt(p, q))).  NaN and +-Inf propagate as IEEE addition does.
 * Backward: dx[n][h][w][c] = the sum of float(dy[n][p][q][c]) / float(cnt(p, q)) over the windows (p, q) that contain (h, w), in
 *   ascending p, then ascending q, each quotient rounded, the sum starting from the first term and rounded to bf16 once; +0 with
 *   no term.  Every element of dx is written, with no memset and no atomics.
 * The pad columns and pad rows of y's layout are never written; those of dy are never read.  x and y disjoint, dy and dx
 * disjoint, every pointer 16-byte aligned.  Stream-ordered, no allocation, the same bits on every run and SM count.
 * pcnn_avgpool_nhwc_info: host only, out5 as pcnn_maxpool_nhwc_info. */
int pcnn_avgpool_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, void *y_bf16_dev, int N, int H, int W, int C, int R, int S,
                               int stride, int pad_h, int pad_w, int count_include_pad, int y_row_pitch, int y_image_rows);
int pcnn_avgpool_nhwc_bf16_bwd(pcnn_ctx *ctx, const void *dy_bf16_dev, void *dx_bf16_dev, int N, int H, int W, int C, int R, int S,
                               int stride, int pad_h, int pad_w, int count_include_pad, int dy_row_pitch, int dy_image_rows);
int pcnn_avgpool_nhwc_info(int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int row_pitch, int image_rows,
                           int *out5);
/* Global average pooling (csrc/pool_nhwc.cu), as torch.nn.functional.adaptive_avg_pool2d(x, 1) or x.mean((2, 3)):
 *   - x and dx are dense bf16 [N][H][W][C]: what a conv forward or a batch norm writes as y, and what their backward reads as dy;
 *   - y and dy are [N][1][row_pitch], row_pitch 0 = C rounded up to 8, otherwise >= C and a multiple of 8: the x layout of a
 *     LinearLayer with P = Q = 1, so the pool sits between a batch norm and a linear layer with no copy.
 * Forward: s = the sum of float(x[n][h][w][c]) over the H W pixels in fp32, in the order of the partition pcnn_global_avgpool_nhwc_info
 *   reports, which depends on (N, H, W, C) alone, never on the SM count: the pixels are cut into ranges of `pixels per CTA`; in a
 *   range, lane l (0..lanes-1) sums the pixels l, l + lanes, ... from its first one; the lanes holding a pixel are added in lane
 *   order; the ranges of an image are added in range order (through fp32 slots in the context's scratch block when there are
 *   several).  y[n][c] = bf16_rn(s / float(H W)).  The pad columns of y are never written.
 * Backward: dx[n][h][w][c] = bf16_rn(float(dy[n][c]) / float(H W)) for every pixel; the pad of dy is never read.
 * Domain (anything else is PCNN_ERR_ARG with the function and the rule in the message): N, H, W, C >= 1; H W C within the 32-bit
 * index range of one image; the row pitch above; every pointer 16-byte aligned; x and y, dy and dx disjoint.  Channel groups (8
 * channels when C % 8 == 0, else 1) beyond 256 are sliced across CTAs.  Stream-ordered; the same bits on every run and SM count.
 * pcnn_global_avgpool_nhwc_info: host only (no GPU, no context).  out8 = { row pitch used, channels per thread (8 or 1), channel
 * groups per CTA, channel slices, pixel lanes per CTA, pixels per CTA (8 per lane), pixel ranges per image, CTAs of the forward }. */
int pcnn_global_avgpool_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, void *y_bf16_dev, int N, int H, int W, int C, int y_row_pitch);
int pcnn_global_avgpool_nhwc_bf16_bwd(pcnn_ctx *ctx, const void *dy_bf16_dev, void *dx_bf16_dev, int N, int H, int W, int C,
                                      int dy_row_pitch);
int pcnn_global_avgpool_nhwc_info(int N, int H, int W, int C, int row_pitch, int *out8);
/* Batch normalization between convolution layers (csrc/batchnorm_nhwc.cu), as torch.nn.functional.batch_norm with affine
 * parameters, followed by an optional residual add and ReLU, SiLU, hard-swish or ReLU6.  x, r, y, dy, dy2, dx and dr are dense bf16 [pixels][C] (pixels =
 * N H W: the layout both conv forwards write as y and the gradients read as dy); gamma, beta, the running and the saved
 * statistics, dgamma and dbeta are fp32 [C].  M = pixels.  Every fp32 operation below rounds to nearest with no contraction.
 * Forward, training = 1:
 *   - mean and the biased variance var of float(x) over the M pixels of each channel, accumulated so that a mean large next to
 *     the spread does not cancel (per-CTA sums of x - k in fp32, k the CTA's first pixel, merged in double in a fixed order;
 *     not E[x^2] - E[x]^2): save_mean = float(mean), save_rstd = float(1 / sqrt(var + double(eps))) in double;
 *   - when running_mean and running_var are given (both or neither): with keep = 1 - momentum in fp32,
 *       running_mean = keep * running_mean + momentum * save_mean
 *       running_var  = keep * running_var + momentum * float(var * M / (M - 1))   (the unbiased variance, as torch)
 *     each product rounded, then the sum.
 * Forward, training = 0: mean = running_mean and rstd = float(1 / sqrt(double(running_var) + double(eps))) in double; nothing
 * but y is written (save_mean, save_rstd and momentum are not used).
 * Then per element, with mean and rstd those of the channel:
 *   xhat = (float(x) - mean) * rstd;  v = xhat * gamma + beta;  v = v + float(r) when r is given;
 *   y = bf16_rn(act(v)), act 0 none or 3 the ReLU of the conv epilogues (v < 0 ? +0 : v, NaN and -0 unchanged), or one of
 *   the activations of EfficientNet, MobileNetV3 and MobileNetV2 (RN = fp32 round to nearest, "/" the IEEE quotient):
 *     4 SiLU:       RN(v / RN(1 + E(-v)))                                     (torch: x / (1 + exp(-x)))
 *     5 hard-swish: RN(RN(v * u) / 6), u = min(max(RN(v + 3), 0), 6)          (torch: x * min(max(x + 3, 0), 6) / 6)
 *     6 ReLU6:      min(max(v, 0), 6) as v < 0 ? +0 : (v > 6 ? 6 : v)          (torch: hardtanh(x, 0, 6))
 *   with NaN passing every min / max (NaN in, NaN out) and -0 kept by ReLU6, as torch.  Where fp32 departs from torch's
 *   float64: SiLU gives -0 for v < -88.7228317 (E(-v) = +Inf; the exact value is below 2^-119 in magnitude) and NaN at v = -Inf
 *   (as torch); hard-swish gives +Inf for v > FLT_MAX / 6 (RN(v * 6) overflows) and NaN at v = -Inf (as torch).
 *   E(x) is the library's exponential, a fixed sequence of fp32 operations a numpy float32 replay reproduces bit for bit
 *   (expf and __expf cannot be replayed):
 *     x > 88.7228317 (0x42B17217) -> +Inf;  x < -103.972076 (0xC2CFF1B4) -> +0;  NaN -> NaN;  otherwise
 *     k = rint(RN(x * log2e)), log2e = 0x3FB8AA3B;
 *     r = RN(RN(x - RN(k * ln2_hi)) - RN(k * ln2_lo)), ln2_hi = 0x3F317200 (15 significant bits: k * ln2_hi and x - k * ln2_hi
 *       are exact), ln2_lo = 0x35BFBE8E;
 *     p = c6, then p = RN(RN(p * r) + c_i) for i = 5 .. 0 (Horner), c0 = c1 = 1, c2 = 0x3EFFFFFE, c3 = 0x3E2AAA0C,
 *       c4 = 0x3D2AAC12, c5 = 0x3C0933ED, c6 = 0x3AB5736C (a minimax fit on |r| <= ln2 / 2);
 *     E = RN(RN(p * 2^k1) * 2^k2), k1 = floor(k / 2), k2 = k - k1: the first product is exact, so a subnormal result is rounded
 *       once and a result near FLT_MAX overflows only when it should.
 *   Its error over the finite inputs is at most 1.30 ulp of exp(x) (measured 1.2965 at every 97th bit pattern, the thresholds
 *   and the subnormal results; 99.5 % correctly rounded).
 * Act 1 is refused: the sigmoid of the conv epilogues uses tanh.approx, which no reference can replay bit for bit.
 * Backward (of a training forward; save_mean and save_rstd are what it wrote, y its output):
 *   t = float(dy), or float(dy) + float(dy2) when dy2 (a second gradient arriving at a residual join) is given;
 *   g = bf16_rn(act'(t)): at act 3 float(y) <= 0 gives +0 (a NaN y passes t), as threshold_backward; without dy2 dy's bits pass;
 *   dbeta = sum over pixels of float(g), dgamma = sum of float(g) * xhat (xhat exactly as in the forward), in fp32 per-CTA
 *     partials over pixel ranges that depend only on (pixels, C), then a fixed-order pass over them;
 *   dx = bf16_rn(((float(g) - dbeta / Mf) - xhat * (dgamma / Mf)) * (gamma * rstd)), Mf = float(M), the two quotients and
 *     gamma * rstd formed once per channel from the dgamma and dbeta just written;
 *   dr = g when dr is given: the gradient of the residual input r.
 * Backward at codes 4-6 (pcnn_batchnorm_nhwc_bf16_bwd_preact; pcnn_batchnorm_nhwc_bf16_bwd refuses them, and this entry refuses
 * 0 and 3, so each code has one backward): y cannot give the derivative (SiLU and hard-swish are not monotonic, and bf16 rounds
 * every v in (5.984, 6) to a ReLU6 y of 6), so each pass recomputes v from x, save_mean, save_rstd, gamma, beta and r exactly as
 * the forward formed it (r must be the forward's r, unchanged, or NULL if it had none), and with t as above
 *     4 SiLU:       s = RN(1 / RN(1 + E(-v))), d = RN(s * RN(1 + RN(v * RN(1 - s)))), g = bf16_rn(RN(t * d))
 *                   (torch's silu_backward multiplies t * s first; the float64 results agree)
 *     5 hard-swish: v <= -3 -> +0;  v >= 3 -> t passes;  otherwise g = bf16_rn(RN(t * RN(RN(v / 3) + 0.5)))  (hardswish_backward;
 *                   NaN gives NaN, as torch's vectorised loop; its scalar tail passes t)
 *     6 ReLU6:      0 < v < 6 -> t passes;  otherwise +0, NaN included  (hardtanh_backward)
 *   where a passed t is bf16_rn(t) (dy's bits without dy2).  dbeta, dgamma, dx and dr then follow the rules above with this g.
 * dx == dy (in place) is allowed; no other two buffers may overlap.  Domain (anything else is PCNN_ERR_ARG with the function and
 * the rule in the message; the shape rules read the same in pcnn_batchnorm_nhwc_info):
 *   - 1 <= C <= 256; training 0 or 1; M >= 2 when training and for the backward, M >= 1 in eval;
 *   - eps finite and >= 0; 0 <= momentum <= 1; act 0, 3, 4, 5 or 6 in the forward, 0 or 3 in pcnn_batchnorm_nhwc_bf16_bwd, 4, 5
 *     or 6 in pcnn_batchnorm_nhwc_bf16_bwd_preact (which also needs beta; r, dy2 and dr may be NULL);
 *   - every pointer 16-byte aligned; x, y, gamma, beta not NULL; save_mean and save_rstd not NULL when training; running_mean
 *     and running_var not NULL in eval; x, y, dy, gamma, the saved statistics, dx, dgamma and dbeta not NULL in the backward.
 * With C % 8 == 0 the passes move 16-byte vectors of 8 channels, otherwise single elements.  No atomics: reruns and every H100
 * give the same bits.  Elements past pixels * C are never written.  All calls are stream-ordered and use the context's one
 * scratch block for their per-CTA partials.
 * pcnn_batchnorm_nhwc_info: host only (no GPU, no context).  out5 = { channels per thread (8 or 1), pixel lanes per CTA, pixels
 * per CTA, slots of the statistics pass (0 when training = 0), slots of the gradient pass }. */
int pcnn_batchnorm_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, const void *r_bf16_dev, void *y_bf16_dev, long pixels, int C,
                                 int act, int training, float eps, float momentum, const float *gamma_dev, const float *beta_dev,
                                 float *running_mean_dev, float *running_var_dev, float *save_mean_dev, float *save_rstd_dev);
int pcnn_batchnorm_nhwc_bf16_bwd(pcnn_ctx *ctx, const void *x_bf16_dev, const void *y_bf16_dev, const void *dy_bf16_dev,
                                 const void *dy2_bf16_dev, const float *gamma_dev, const float *save_mean_dev, const float *save_rstd_dev,
                                 void *dx_bf16_dev, void *dr_bf16_dev, float *dgamma_dev, float *dbeta_dev, long pixels, int C, int act);
int pcnn_batchnorm_nhwc_bf16_bwd_preact(pcnn_ctx *ctx, const void *x_bf16_dev, const void *r_bf16_dev, const void *dy_bf16_dev,
                                        const void *dy2_bf16_dev, const float *gamma_dev, const float *beta_dev, const float *save_mean_dev,
                                        const float *save_rstd_dev, void *dx_bf16_dev, void *dr_bf16_dev, float *dgamma_dev,
                                        float *dbeta_dev, long pixels, int C, int act);
int pcnn_batchnorm_nhwc_info(long pixels, int C, int training, int *out5);
/* Group normalization between convolution layers (csrc/groupnorm_nhwc.cu), as torch.nn.functional.group_norm(x, G, gamma, beta,
 * eps), followed by batch normalization's optional residual add and activation.  x, r, y, dy, dy2, dx and dr are dense bf16
 * [N][HW][C] (the layout both conv forwards write as y); gamma, beta, dgamma and dbeta are fp32 [C]; save_mean and save_rstd are
 * fp32 [N][G]; dstat is fp32 [2][N][G].  Cg = C / G; group g of image n is the channels [g Cg, (g + 1) Cg) over all HW pixels,
 * Mg = HW Cg elements, Mgf = float(Mg).  With G = C this is instance normalization with affine parameters, with G = 1 layer
 * normalization over (C, H, W) with per-channel parameters.  There are no running statistics: training and evaluation compute the
 * same y.  Every fp32 operation below rounds to nearest with no contraction.
 * Forward:
 *   - mean and the biased variance var of float(x) over each (n, g), accumulated so that a mean large next to the spread does not
 *     cancel (fp32 sums of x - k per image, channel and pixel range, k the range's first pixel of that channel, merged in double
 *     in a fixed order; not E[x^2] - E[x]^2): save_mean = float(mean), save_rstd = float(1 / sqrt(var + double(eps))) in double;
 *   - per element, with mean and rstd those of the element's (n, g): xhat = (float(x) - mean) * rstd;  v = xhat * gamma[c] +
 *     beta[c];  v = v + float(r) when r is given;  y = bf16_rn(act(v)), act 0, 3, 4, 5 or 6 exactly as in
 *     pcnn_batchnorm_nhwc_bf16_fwd (act 1 is refused for the reason given there).
 * Backward at codes 0 and 3 (pcnn_groupnorm_nhwc_bf16_bwd, of a forward whose save_mean and save_rstd it wrote and whose output was
 * y) and at codes 4-6 (pcnn_groupnorm_nhwc_bf16_bwd_preact, which recomputes v from x, the saved statistics, gamma, beta and r as
 * the forward formed it; r must be the forward's r, unchanged, or NULL if it had none).  Each entry refuses the other's codes.
 *   t and g = bf16_rn(act'(t)) are batch normalization's, per element;
 *   dbeta[c] = sum of float(g), dgamma[c] = sum of float(g) * xhat, each over all N HW pixels (fp32 per-CTA partials over pixel
 *     ranges, then a fixed-order pass over them);
 *   A[n][g] = sum of gamma[c] * float(g), B[n][g] = sum of gamma[c] * float(g) * xhat, each over the Mg elements of the group: the
 *     per-channel fp32 partials of the pixel ranges times gamma[c], added in double in a fixed order, then rounded to float and
 *     written to dstat[0][n][g] and dstat[1][n][g];
 *   dx = bf16_rn(RN(RN(RN(RN(float(g) * gamma[c]) - a) - RN(xhat * b)) * rstd)), a = RN(A / Mgf) and b = RN(B / Mgf) formed once
 *     per (n, g) from the dstat just written, so dx is a stated function of x, g, the saved statistics, gamma and dstat;
 *   dr = g when dr is given: the gradient of the residual input r.
 * Partition: the pixel ranges of an image (of `pixels per range` each) and the channel slices (at most 256 channels) depend on
 * (HW, C, G) alone, never on N.  So an image's y, save_mean, save_rstd, dstat, dx and dr are bit-identical whether it runs alone
 * or at any position of any batch; dgamma and dbeta, sums over the batch, are not.
 * dx == dy (in place) is allowed; no other two buffers may overlap.  Domain (anything else is PCNN_ERR_ARG with the function and
 * the rule in the message; the shape rules read the same in pcnn_groupnorm_nhwc_info):
 *   - N >= 1; HW >= 1; 1 <= C <= 2048; 1 <= G <= C with C % G == 0; N * ranges * slices < 2^31 CTAs;
 *   - eps finite and >= 0; act 0, 3, 4, 5 or 6 in the forward, 0 or 3 in pcnn_groupnorm_nhwc_bf16_bwd, 4, 5 or 6 in
 *     pcnn_groupnorm_nhwc_bf16_bwd_preact;
 *   - every pointer 16-byte aligned; only r may be NULL in the forward; only dy2 and dr in pcnn_groupnorm_nhwc_bf16_bwd (dstat
 *     is required); only r, dy2 and dr in pcnn_groupnorm_nhwc_bf16_bwd_preact (beta and dstat are required).
 * With C % 8 == 0 the passes move 16-byte vectors of 8 channels (which may span several groups when Cg < 8), otherwise single
 * elements.  No atomics: reruns and every H100 give the same bits.  Elements past N HW C are never written.  All calls are
 * stream-ordered and use the context's one scratch block for their per-CTA partials.
 * pcnn_groupnorm_nhwc_info: host only (no GPU, no context).  out11 = { channels per thread (8 or 1), channel groups of that width
 * per CTA, channel slices, pixel lanes per CTA, pixels per range, ranges per image, CTAs of each elementwise pass (N x ranges x
 * slices: the statistics, y, the gradient sums and dx), slots per channel (N x ranges), CTAs of the two per-(n, g) merges (8 pairs
 * each), n_acc of dgamma and dbeta, n_acc of A, B and the statistics }.  n_acc is the number of fp32 roundings on the longest
 * path of one sum: a bound of 2 n_acc 2^-24 sum |terms| holds. */
int pcnn_groupnorm_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, const void *r_bf16_dev, void *y_bf16_dev, int N, int HW, int C,
                                 int G, int act, float eps, const float *gamma_dev, const float *beta_dev, float *save_mean_dev,
                                 float *save_rstd_dev);
int pcnn_groupnorm_nhwc_bf16_bwd(pcnn_ctx *ctx, const void *x_bf16_dev, const void *y_bf16_dev, const void *dy_bf16_dev,
                                 const void *dy2_bf16_dev, const float *gamma_dev, const float *save_mean_dev, const float *save_rstd_dev,
                                 void *dx_bf16_dev, void *dr_bf16_dev, float *dgamma_dev, float *dbeta_dev, float *dstat_dev, int N, int HW,
                                 int C, int G, int act);
int pcnn_groupnorm_nhwc_bf16_bwd_preact(pcnn_ctx *ctx, const void *x_bf16_dev, const void *r_bf16_dev, const void *dy_bf16_dev,
                                        const void *dy2_bf16_dev, const float *gamma_dev, const float *beta_dev, const float *save_mean_dev,
                                        const float *save_rstd_dev, void *dx_bf16_dev, void *dr_bf16_dev, float *dgamma_dev,
                                        float *dbeta_dev, float *dstat_dev, int N, int HW, int C, int G, int act);
int pcnn_groupnorm_nhwc_info(int N, int HW, int C, int G, int *out11);
/* ---- self-attention ---------------------------------------------------------------------------------------------------------
 * Self-attention over the T = H W pixels of each image (csrc/attention_tc.cu), as torch's scaled_dot_product_attention without a
 * mask or dropout: per image n and head j, O = softmax(scale Q K^T) V.  q, k and v are bf16 with element (n, t, head j, i) at
 * (n T + t) ld + j d + i, one ld for all three: with a fused qkv projection [N T][3 h d] they are its columns 0, h d and 2 h d, and
 * ld = 3 h d.  o and dout are dense bf16 [N][T][h][d] (the x and dy of an output projection); lse is fp32 [N][h][T]; dq, dk and dv
 * are written in q's layout with rows of ld_g elements, so the fused projection's dy is written in place.
 * Forward, per row (image, head, query t), over key blocks of 64 in order; fp32 rounds to nearest without contraction:
 *   1. scores s = q . k in fp32 on the tensor cores (bf16 products exact, fp32 accumulation in an order the hardware fixes);
 *   2. u = RN(s c2), c2 = float(scale log2 e); keys >= T are u = -inf;
 *   3. running max m = max(m, the block's u) (exact);
 *   4. exponent p = ex2.approx(RN(u - m)) (relative error below 2^-22), alpha = ex2.approx(RN(m_old - m)) rescales l and acc;
 *   5. P = bf16_rn(p);
 *   6. sum l = RN(RN(l alpha) + the block's sum of P in fp32);
 *   7. acc = RN(acc alpha) + P V in fp32 on the tensor cores;
 *   8. division: o = bf16_rn(RN(acc RN(1 / l)));
 *   9. lse = RN(RN(m + lg2.approx(l)) ln 2) (lg2.approx: absolute error below 2^-21), the natural-log logsumexp of scale s.
 * Backward (pcnn_attention_bf16_bwd, given the forward's o and lse):
 *   - D = sum over i of float(dout) float(o) per row, fp32 fma in the order i = 0 .. d - 1 (into the context's scratch);
 *   - P = ex2.approx(RN(RN(s c2) - RN(lse log2 e))) recomputed, 0 for keys (dQ) or queries (dK, dV) >= T; dP = dout . v in fp32;
 *   - dS = bf16_rn(RN(P RN(dP - D))), from the fp32 P; dV = bf16_rn(sum over queries of bf16_rn(P) dout) in fp32;
 *   - scale placement: dQ = bf16_rn(RN(scale (sum over keys of dS k))) and dK = bf16_rn(RN(scale (sum over queries of dS q))),
 *     the scale applied once, to the fp32 sums.
 * Partition: a tile is (image, head, block of 128 query rows) in the forward and dQ kernels and (image, head, block of 128 keys) in
 * the dK/dV kernel; each loops over blocks of 64 in a fixed order, with no atomics.  So the bits of one (image, head) do not depend
 * on N, the other heads, the SM count or the run.  Rows past T, the columns of other heads and everything past the last row of a
 * buffer are never written.
 * Domain (anything else is PCNN_ERR_ARG with the called function and the rule in the message; the shape rules read the same in
 * pcnn_attention_info):
 *   - d 16, 32, 64 or 128; heads >= 1; N >= 1; 1 <= T <= 16384; N heads ceil(T / 128) tiles < 2^31;
 *   - ld and ld_g >= heads d and multiples of 8; scale finite and > 0;
 *   - every pointer 16-byte aligned; dq, dk and dv may share a buffer on disjoint columns; no output overlaps an input or
 *     another output otherwise.
 * pcnn_attention_info: host only (no GPU, no context), with ld_g 0 for the forward's rules alone.  out8 = { query rows per tile,
 * rows per streamed block, stages, tiles of the forward, of the dK/dV kernel and of the dQ kernel, scratch bytes of the backward,
 * dynamic shared memory of a backward kernel }. */
int pcnn_attention_bf16_fwd(pcnn_ctx *ctx, const void *q_bf16_dev, const void *k_bf16_dev, const void *v_bf16_dev, int N, int T, int heads,
                            int d, int ld, float scale, void *o_bf16_dev, float *lse_dev);
int pcnn_attention_bf16_bwd(pcnn_ctx *ctx, const void *q_bf16_dev, const void *k_bf16_dev, const void *v_bf16_dev, const void *o_bf16_dev,
                            const void *dout_bf16_dev, const float *lse_dev, int N, int T, int heads, int d, int ld, float scale,
                            void *dq_bf16_dev, void *dk_bf16_dev, void *dv_bf16_dev, int ld_g);
int pcnn_attention_info(int N, int T, int heads, int d, int ld, int ld_g, float scale, long long *out8);
/* Fully connected layers (csrc/linear_tc.cu), bf16 on the tensor cores with fp32 accumulation:
 *   - x is [N][image_rows][row_pitch] bf16 with P x Q pixels of C channels per image: the layout a plan reads as x and the NHWC
 *     pool writes as y.  A previous linear layer's y is the same with P = Q = 1, C = its O, row_pitch = O, image_rows 1.
 *   - F = P Q C features in NHWC order; W fp32 [O][P][Q][C] (KRSC with K = O, R = P, S = Q), b fp32 [O];
 *   - y, dy are dense bf16 [N][O]; dW is fp32 [O][P][Q][C].
 * pcnn_linear_plan_create returns a pcnn_conv_plan: pcnn_conv_tc_fwd runs it, y[n][o] = act(b[o] + sum_f x[n][f] W[o][f]) (the
 * activations of the conv forwards, PCNN_ACT_*), pcnn_conv_plan_set_params refreshes W (fp32 [O][P][Q][C]) and b from device memory, and
 * pcnn_conv_tc_plan_destroy frees it.  The plan holds W rounded to bf16 (round to nearest even, on the device).
 * pcnn_linear_wgrad: dW[o][f] = sum_n dy[n][o] x[n][f], fp32.  pcnn_linear_dgrad: dx[n][f] = sum_o dy[n][o] Wbf16[o][f], rounded to
 * bf16 once, written in x's layout: exactly the dy pcnn_maxpool_nhwc_bf16_bwd reads, or a previous linear layer's dy.  dx uses the
 * plan's bf16 weights, the bits the forward multiplied: call it before pcnn_conv_plan_set_params.  Both take the shape from the
 * plan; a plan not made by pcnn_linear_plan_create is PCNN_ERR_ARG.
 * Pad columns and pad rows of x are never read (NaN there changes no bit); those of dx are never written; y and dx rows of
 * every image are fully written.  Reductions may be split into ranges whose fp32 partials are added in a fixed order; the
 * split depends on the shape only, so reruns and every H100 give the same bits.  All calls are stream-ordered.
 * Domain (anything else is PCNN_ERR_ARG with the rule in the message, the same for the create call and the query):
 *   - N, P, Q, C >= 1, 1 <= O <= 256 (the limit of pcnn_conv_bias_act_bwd, which serves as the layer's bias / activation backward);
 *   - F <= 2^24;
 *   - row_pitch 0 = Q C rounded up to a multiple of 8, otherwise >= Q C and a multiple of 8 (so a hidden width that feeds another
 *     linear layer must be a multiple of 8); image_rows 0 = P, otherwise >= P;  act 0 (none), 1 (sigmoid) or 3 (ReLU);
 *   - every device pointer 16-byte aligned.
 * pcnn_linear_info: host only (no GPU, no context).  out12 = { row pitch used, 128-image tiles, forward reduction steps (64-feature
 * chunks), forward splits, forward stages, weight-gradient chunk pairs, weight-gradient splits (image ranges), weight-gradient
 * stages, input-gradient tiles, chunks per input-gradient tile, input-gradient stages, forward MMA width (O rounded up to 16) }. */
int pcnn_linear_plan_create(pcnn_ctx *ctx, int N, int P, int Q, int C, int O, int row_pitch, int image_rows, int act,
                            const float *w_host, const float *b_host, pcnn_conv_plan **out);
int pcnn_linear_wgrad(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *x_bf16_dev, const void *dy_bf16_dev, float *dw_f32_dev);
int pcnn_linear_dgrad(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *dy_bf16_dev, void *dx_bf16_dev);
int pcnn_linear_info(int N, int P, int Q, int C, int O, int row_pitch, int image_rows, int *out12);
/* Depthwise convolution (csrc/dwconv_nhwc.cu), as torch.nn.functional.conv2d(x, w, b, stride, padding=(pad_h, pad_w), groups=C)
 * with w [C][1][R][S]: each channel is filtered by its own R x S filter.
 *   - x and dx are dense bf16 [N][H][W][C], y and dy dense bf16 [N][P][Q][C]: what the conv forwards and batch norm write and
 *     what batch norm, the global average pool and pcnn_conv_bias_act_bwd read;
 *     P = (H + 2 pad_h - R) / stride + 1,   Q = (W + 2 pad_w - S) / stride + 1;
 *   - filters fp32 [C][R][S] (KRSC with one input channel: torch's weight reshaped), bias fp32 [C], dw fp32 [C][R][S].
 * pcnn_dwconv_plan_create returns a pcnn_conv_plan: pcnn_conv_tc_fwd runs it, pcnn_conv_plan_set_params refreshes its filters and
 * bias from device memory, pcnn_optim_step refreshes them with the update, and pcnn_conv_tc_plan_destroy frees it.  The plan holds
 * the filters rounded to bf16 (round to nearest even, on the device) in the master's [C][R][S] order.
 * Rules (fp32 round to nearest; every product float(bf16) * float(bf16) is exact in fp32, so an FMA gives the bits of a product
 * followed by an add).  The window of output (p, q) starts at (h0, w0) = (p stride - pad_h, q stride - pad_w); a tap outside the
 * image reads x = +0 and is multiplied like any other (0 * Inf is NaN), as torch does.
 *   Forward: acc = the sum over r = 0..R-1, then s = 0..S-1, of float(x[n][h0 + r][w0 + s][c]) * float(wbf16[c][r][s]), starting
 *     from the first term; v = acc + b[c] with a bias; y = bf16_rn(act(v)), act 0 (none) or 3 (the ReLU of the conv epilogues:
 *     v < 0 ? +0 : v, NaN and -0 unchanged).  Act 1 is refused: the sigmoid uses tanh.approx, which no reference can replay.
 *   Input gradient: dx[n][h][w][c] = the sum of float(dy[n][p][q][c]) * float(wbf16[c][r][s]) over the taps with h = p stride -
 *     pad_h + r and w = q stride - pad_w + s for some 0 <= p < P, 0 <= q < Q, in ascending r, then ascending s, starting from the
 *     first term, rounded to bf16 once; +0 with no term.  Every element of dx is written, with no memset and no atomics.  It uses
 *     the plan's bf16 filters, the bits the forward multiplied: call it before the filters are refreshed.
 *   Weight gradient: dw[c][r][s] = the sum over n, p, q of float(dy[n][p][q][c]) * float(x~[n][h0 + r][w0 + s][c]) (x~ = +0 outside
 *     the image).  The N P Q output pixels are cut into ranges of `pixels per range` (a function of the shape alone, never of the SM
 *     count); in a range, lane l sums the pixels l, l + lanes, ... from its first one, the lanes holding a pixel are added in lane
 *     order, and with several ranges each range writes an fp32 slot in the context's scratch block which
 *     pcnn_conv_wgrad_reduce_slots adds in a fixed order.  dw is overwritten, not accumulated.
 * Both gradients take the shape from the plan; a plan not made by pcnn_dwconv_plan_create is PCNN_ERR_ARG.  All calls are
 * stream-ordered and give the same bits on every run and SM count.
 * Domain (anything else is PCNN_ERR_ARG with the function and the rule in the message; pcnn_dwconv_info makes the create call's
 * refusals):
 *   - N, H, W, C >= 1 (C has no upper limit); 1 <= R, S <= 7; stride 1..4;
 *   - 0 <= pad_h <= R - 1, 0 <= pad_w <= S - 1, H + 2 pad_h >= R and W + 2 pad_w >= S;
 *   - H W C, P Q C and C R S within the 32-bit index range;  act 0 or 3;
 *   - every pointer 16-byte aligned; x and y disjoint, dy and dx disjoint, dw disjoint from x and dy.
 * With C % 8 == 0 the passes move 16-byte vectors of 8 channels, otherwise single elements.
 * pcnn_dwconv_info: host only (no GPU, no context).  out9 = { P, Q, channels per thread (8 or 1), channel groups per CTA, channel
 * slices, weight-gradient pixel lanes per range, pixels per range, ranges, n_acc: the fp32 additions on the longest path of one
 * dw sum (pixels of a lane - 1, lanes - 1, and with several ranges ceil(ranges / 8) + 3 in pcnn_conv_wgrad_reduce_slots) }. */
int pcnn_dwconv_plan_create(pcnn_ctx *ctx, int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int act,
                            const float *filt_host, const float *bias_host, pcnn_conv_plan **out);
int pcnn_dwconv_wgrad(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *x_bf16_dev, const void *dy_bf16_dev, float *dw_f32_dev);
int pcnn_dwconv_dgrad(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *dy_bf16_dev, void *dx_bf16_dev);
int pcnn_dwconv_info(int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int *out9);
/* The same depthwise convolution with a dilation (dil_h, dil_w), as conv2d(..., dilation=(dil_h, dil_w), groups=C): tap (r, s)
 * of the window of output (p, q) reads x~[n][h0 + r dil_h][w0 + s dil_w][c].  With E_h = dil_h (R - 1) + 1, E_w = dil_w (S - 1) + 1,
 *     P = (H + 2 pad_h - E_h) / stride + 1,   Q = (W + 2 pad_w - E_w) / stride + 1,
 * and every rule above holds with r dil_h for r and s dil_w for s: the forward sums over ascending r, then s; the input gradient
 * takes the taps with h = p stride - pad_h + r dil_h and w = q stride - pad_w + s dil_w in ascending r, then s (+0 with no term);
 * the weight gradient's lanes, ranges and slot reduction are unchanged.  The plan is an ordinary depthwise plan: pcnn_conv_tc_fwd,
 * pcnn_dwconv_wgrad, pcnn_dwconv_dgrad, pcnn_conv_plan_set_params and pcnn_optim_step take it as they take one of
 * pcnn_dwconv_plan_create.  The domain is the one above with, in place of its padding and fit rules,
 *   - 1 <= dil_h, dil_w <= 256;
 *   - 0 <= pad_h <= dil_h (R - 1), 0 <= pad_w <= dil_w (S - 1), H + 2 pad_h >= E_h and W + 2 pad_w >= E_w.
 * At dilation (1, 1) each is exactly pcnn_dwconv_plan_create / pcnn_dwconv_info, refusals and their text included, except that
 * refusals name the called function.  out9 as pcnn_dwconv_info's. */
int pcnn_dwconv_plan_create_dilated(pcnn_ctx *ctx, int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int dil_h,
                                    int dil_w, int act, const float *filt_host, const float *bias_host, pcnn_conv_plan **out);
int pcnn_dwconv_info_dilated(int N, int H, int W, int C, int R, int S, int stride, int pad_h, int pad_w, int dil_h, int dil_w, int *out9);
/* Grouped convolution (csrc/gconv_nhwc.cu), as torch.nn.functional.conv2d(x, w, b, stride, padding=(pad_h, pad_w), groups=G) with
 * w [K][Cg][R][S], 1 < G: each group g of Cg = C / G input channels feeds its own Kg = K / G filters; output k belongs to group
 * g = k / Kg (ResNeXt, RegNet, ShuffleNet, and a depthwise layer with a channel multiplier: Cg = 1, Kg > 1).
 *   - x and dx are dense bf16 [N][H][W][C], y and dy dense bf16 [N][P][Q][K]: the layouts of the conv forwards, batch norm and the
 *     global average pool; P = (H + 2 pad_h - R) / stride + 1,   Q = (W + 2 pad_w - S) / stride + 1;
 *   - filters fp32 [K][R][S][Cg] (KRSC with the group's Cg input channels: torch's weight permuted), bias fp32 [K], dw fp32
 *     [K][R][S][Cg].
 * pcnn_gconv_plan_create returns a pcnn_conv_plan: pcnn_conv_tc_fwd runs it, pcnn_conv_plan_set_params refreshes its filters and
 * bias from device memory, pcnn_optim_step refreshes them with the update, and pcnn_conv_tc_plan_destroy frees it.  The plan holds
 * the filters rounded to bf16 (round to nearest even, on the device) in the master's [K][R][S][Cg] order, as one row.
 * Rules (fp32 round to nearest; every product float(bf16) * float(bf16) is exact in fp32, so an FMA gives the bits of a product
 * followed by an add).  The window of output (p, q) starts at (h0, w0) = (p stride - pad_h, q stride - pad_w); a tap outside the
 * image reads x = +0 and is multiplied like any other (0 * Inf is NaN), as torch does.
 *   Forward: acc = the sum over r = 0..R-1, then s = 0..S-1, then c = 0..Cg-1, of float(x[n][h0 + r][w0 + s][g Cg + c]) *
 *     float(wbf16[k][r][s][c]), starting from the first term; v = acc + b[k] with a bias; y = bf16_rn(act(v)), act 0 (none) or 3
 *     (the ReLU of the conv epilogues: v < 0 ? +0 : v, NaN and -0 unchanged).  Act 1 is refused: the sigmoid uses tanh.approx, which
 *     no reference can replay.
 *   Input gradient: dx[n][h][w][g Cg + c] = the sum of float(dy[n][p][q][g Kg + k]) * float(wbf16[g Kg + k][r][s][c]) over the taps
 *     with h = p stride - pad_h + r and w = q stride - pad_w + s for some 0 <= p < P, 0 <= q < Q, in ascending r, then ascending s,
 *     then ascending k = 0..Kg-1, starting from the first term, rounded to bf16 once; +0 with no term.  Every element of dx is
 *     written, with no memset and no atomics.  It uses the plan's bf16 filters, the bits the forward multiplied: call it before the
 *     filters are refreshed.
 *   Weight gradient: dw[k][r][s][c] = the sum over n, p, q of float(dy[n][p][q][k]) * float(x~[n][h0 + r][w0 + s][g Cg + c]) (x~ = +0
 *     outside the image).  The N P Q output pixels are cut into ranges of `pixels per range` (a function of the shape alone, never of
 *     the SM count); in a range, lane l of `lanes` sums the pixels l, l + lanes, ... from its first one, the lanes holding a pixel are
 *     added in lane order, and with several ranges each range writes an fp32 slot in the context's scratch block which
 *     pcnn_conv_wgrad_reduce_slots adds in a fixed order.  dw is overwritten, not accumulated.
 * Both gradients take the shape from the plan; a plan not made by pcnn_gconv_plan_create is PCNN_ERR_ARG, and the other plan kinds'
 * gradient calls refuse a grouped plan.  All calls are stream-ordered and give the same bits on every run and SM count.
 * Domain (anything else is PCNN_ERR_ARG with the function and the rule in the message; pcnn_gconv_info makes the create call's
 * refusals):
 *   - the window rules of the depthwise convolution: N, H, W, C >= 1; 1 <= R, S <= 7; stride 1..4; 0 <= pad_h <= R - 1,
 *     0 <= pad_w <= S - 1, H + 2 pad_h >= R and W + 2 pad_w >= S;
 *   - K >= 1; G >= 2 (G = 1, a dense convolution, is refused with a message naming the dense plans); C % G == 0 and K % G == 0;
 *     Cg = Kg = 1 (a depthwise convolution) is refused with a message naming pcnn_dwconv_plan_create; Cg = 1 with Kg > 1 is taken;
 *   - one group's filters Kg Cg R S <= 36864 (72 KiB of bf16: a CTA stages the filters it applies through shared memory), which
 *     admits every 1x1 and 3x3 filter with Cg, Kg <= 64 and every 5x5 and 7x7 with Cg Kg <= 64;
 *   - H W C, P Q K and K R S Cg within the 32-bit index range (C and K have no other limit);  act 0 or 3;
 *   - every pointer 16-byte aligned; x and y disjoint, dy and dx disjoint, dw disjoint from x and dy.
 * Each pass loads vectors of the largest of 8, 4, 2, 1 channels that divides its reduced axis (Cg for the forward and the weight
 * gradient, Kg for the input gradient): Cg % 8 == 0 moves 16-byte vectors of x, any other Cg a narrower path.
 * pcnn_gconv_info: host only (no GPU, no context).  out16 = { P, Q, Cg, Kg, x channels per load (8, 4, 2 or 1: the largest dividing
 * Cg), output channels per forward thread and dy channels per input-gradient load (the largest dividing Kg), forward k tiles per
 * CTA, forward k slices, input-gradient c tiles per CTA, input-gradient c slices, weight-gradient items, weight-gradient item
 * blocks, pixels per range, ranges, n_acc: the fp32 additions on the longest path of one dw sum (pixels of a lane - 1, lanes - 1,
 * and with several ranges ceil(ranges / 8) + 3 in pcnn_conv_wgrad_reduce_slots), weight-gradient pixel lanes per range }. */
int pcnn_gconv_plan_create(pcnn_ctx *ctx, int N, int H, int W, int C, int K, int G, int R, int S, int stride, int pad_h, int pad_w,
                           int act, const float *filt_host, const float *bias_host, pcnn_conv_plan **out);
int pcnn_gconv_wgrad(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *x_bf16_dev, const void *dy_bf16_dev, float *dw_f32_dev);
int pcnn_gconv_dgrad(pcnn_ctx *ctx, pcnn_conv_plan *plan, const void *dy_bf16_dev, void *dx_bf16_dev);
int pcnn_gconv_info(int N, int H, int W, int C, int K, int G, int R, int S, int stride, int pad_h, int pad_w, int *out16);
/* Squeeze-and-excitation channel gating (csrc/se_nhwc.cu): y = act(x * s[n][c] + r), s = sigmoid(fc2(relu(fc1(GAP(x))))) a gate per
 * image and channel, as in SE-ResNet, MnasNet, MobileNetV3 and EfficientNet.  The squeeze branch runs on the existing layers:
 * pcnn_global_avgpool_nhwc_bf16_fwd writes the x of a linear layer, and linear layers with act 3 and act 1 give s.
 *   - x, r, y, dy, dy2, g and dx are dense bf16 [N][H][W][C]: what the conv forwards and batch norm write as y and read as dy;
 *   - s and ds are dense bf16 [N][C]: the y and dy of a linear layer with O = C;
 *   - dpool is bf16 [N][dpool_row_pitch]: the dy of the global average pool (the dx of the squeeze branch's first linear layer);
 *     row pitch 0 = C rounded up to 8, otherwise >= C and a multiple of 8, as pcnn_global_avgpool_nhwc_bf16_bwd.
 * Rules: every fp32 operation rounds to nearest with no contraction (RN below; a bf16 x bf16 product is exact in fp32 but for
 * underflow, and the kernels round it on its own before any add).
 *   Forward: v = RN(float(x) * float(s[n][c])); v = RN(v + float(r)) when r is given; y = bf16_rn(act(v)), act 0 (none) or 3 (the
 *     ReLU of the conv epilogues: v < 0 ? +0 : v, NaN and -0 unchanged).  Act 1 is refused: the sigmoid uses tanh.approx, which no
 *     reference can replay bit for bit.
 *   Gate gradient (before the squeeze branch's backward): t = float(dy), or RN(float(dy) + float(dy2)) when dy2 (a second gradient
 *     arriving at a residual join) is given; g = bf16_rn(act'(t)) as batch norm's backward: at act 3 float(y) <= 0 gives +0 (a NaN y
 *     passes t); without dy2 dy's bits pass.  g is the gradient of r and the input of the input gradient; g == dy (in place) is
 *     allowed.  ds[n][c] = bf16_rn(the fp32 sum of RN(float(g) * float(x)) over the H W pixels), summed in the order of the global
 *     average pool's partition: the pixels cut into ranges of `pixels per CTA`; in a range, lane l sums the pixels l, l + lanes, ...
 *     from its first one; the lanes holding a pixel are added in lane order; the ranges of an image in range order, through fp32
 *     slots in the context's scratch block when there are several.  The partition depends on (N, H, W, C) alone, never on the SM
 *     count; pcnn_se_scale_nhwc_info reports it.  ds is the dy of the sigmoid linear layer that wrote s.
 *   Input gradient (after the squeeze branch's backward has written dpool): dx = bf16_rn(RN(float(g) * float(s[n][c]))) without
 *     dpool; with it dx = bf16_rn(RN(RN(float(g) * float(s[n][c])) + RN(float(dpool[n][c]) / float(H W)))), the quotient being the one
 *     pcnn_global_avgpool_nhwc_bf16_bwd rounds: the squeeze branch's gradient joins in the same pass.  dx == g is allowed.  Every
 *     element of dx is written, with no memset and no atomics; the pad of dpool is never read.
 * Domain (anything else is PCNN_ERR_ARG with the function and the rule in the message): N, H, W, C >= 1 (C has no upper limit);
 * H W C within the 32-bit index range of one image, as the global average pool; act 0 or 3; y not NULL at act 3 in the gate pass;
 * every pointer 16-byte aligned; only g == dy and dx == g may share memory.  With C % 8 == 0 the passes move 16-byte vectors of 8
 * channels, otherwise single elements.  Stream-ordered; elements past the tensors are never written; the same bits on every run
 * and SM count.
 * pcnn_se_scale_nhwc_info: host only (no GPU, no context).  out8 = { channels per thread (8 or 1), channel groups per CTA, channel
 * slices, pixel lanes per CTA, pixels per CTA (8 per lane), pixel ranges per image, CTAs of the gate pass, n_acc: the fp32 additions
 * on the longest path of one ds sum (pixels of a lane - 1, lanes holding a pixel - 1, ranges - 1) }. */
int pcnn_se_scale_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, const void *s_bf16_dev, const void *r_bf16_dev, void *y_bf16_dev,
                                int N, int H, int W, int C, int act);
int pcnn_se_scale_nhwc_bf16_bwd_gate(pcnn_ctx *ctx, const void *x_bf16_dev, const void *y_bf16_dev, const void *dy_bf16_dev,
                                     const void *dy2_bf16_dev, void *g_bf16_dev, void *ds_bf16_dev, int N, int H, int W, int C, int act);
int pcnn_se_scale_nhwc_bf16_bwd_input(pcnn_ctx *ctx, const void *g_bf16_dev, const void *s_bf16_dev, const void *dpool_bf16_dev,
                                      int dpool_row_pitch, void *dx_bf16_dev, int N, int H, int W, int C);
int pcnn_se_scale_nhwc_info(int N, int H, int W, int C, int *out8);
/* Dropout and stochastic depth (csrc/dropout.cu): y = x * m (+ r) with m = 0 for a dropped element and 1 / (1 - p) for a kept one,
 * as torch's dropout (element mode) and the drop path of EfficientNet's residual blocks (per-sample mode: one draw per image).
 *   - x, r and y are bf16 arrays of N rows of row_elems elements, consecutive rows row_pitch elements apart (row_pitch 0 = dense,
 *     otherwise >= row_elems).  A dense NHWC activation is N rows of H W C; a global average pool's output is N rows of C at its
 *     row pitch; a dense linear layer's output [N][O] is N rows of O.  The pad (elements row_elems .. row_pitch - 1 of a row) is
 *     never read or written.
 *   - Index: element j of row n is i = n row_elems + j in element mode (per_sample 0) and i = n in per-sample mode (per_sample 1).
 *     It depends on neither the pitch nor the grid nor the SM count: the same arguments give the same bits on every H100.
 *   - Generator: Philox4x32-10 (Salmon et al., SC'11, as Random123) with key (seed lo, seed hi) and counter (q lo, q hi, call lo,
 *     call hi), q = i >> 2; the draw of element i is output word i & 3.  Element i is dropped iff draw < T, T = the uint32 nearest
 *     to p 2^32 (ties to even; p 2^32 above 2^32 - 1/2 gives 2^32 - 1), so the keep probability is 1 - T / 2^32: one 32-bit draw
 *     per element, as torch.  scale = fp32(1 / (1 - p)) evaluated in double and rounded once.  Both are formed on the host and
 *     reported by pcnn_dropout_bf16_info.  p = 0 gives T = 0 and scale 1, and a kernel without the generator.
 *   - Values, fp32 round to nearest with no contraction: m = dropped ? 0.0f : scale; without r y = bf16_rn(float(x) * m); with r
 *     y = bf16_rn(float(r) + RN(float(x) * m)).  A product rather than a select, as torch's native_dropout: a dropped NaN stays
 *     NaN, a dropped Inf gives NaN, a dropped -x gives -0 (and r + -0 = r).
 *   - Backward: dx is this call on dy with the forward's (seed, call, p, per_sample) and no r.  The gradient of r is dy itself.
 *   - y == x and y == r (in place) are allowed; x, r and y must each be the same buffer or share no byte.
 * Domain (anything else is PCNN_ERR_ARG with the function and the rule in the message): N, row_elems >= 1; row_pitch 0 or
 * >= row_elems; p finite with 0 <= p < 1; per_sample 0 or 1; x and y not NULL; every pointer 16-byte aligned.  With row_elems % 8
 * == 0 and row_pitch % 8 == 0 the kernel moves 16-byte vectors of 8 elements of a row (two Philox calls each in element mode, one
 * in per-sample mode), otherwise single elements.  Stream-ordered; a grid-stride loop whose grid depends on the shape alone.
 * pcnn_dropout_bf16_info: host only (no GPU, no context), refused as the call refuses.  out5 = { T, the bits of scale, elements per
 * vector (8 or 1), the grid (CTAs of 256 threads), elements of the busiest thread }. */
int pcnn_dropout_bf16(pcnn_ctx *ctx, const void *x_bf16_dev, const void *r_bf16_dev, void *y_bf16_dev, int N, int row_elems, int row_pitch,
                      double p, int per_sample, unsigned long long seed, unsigned long long call);
int pcnn_dropout_bf16_info(int N, int row_elems, int row_pitch, double p, int per_sample, long long *out5);
/* Input pipeline (csrc/augment.cu): positions first .. first + N - 1 of an epoch of a uint8 dataset in device memory become one
 * bf16 batch in the x layout of every plan, plus its labels, in one launch: a per-epoch shuffle, torchvision's
 * RandomCrop(size = (H, W), padding = pad, fill = 0) and RandomHorizontalFlip on the uint8 image, then ToTensor and
 * Normalize(mean, std).
 *   - Layouts: images dense [n][H][W][C] uint8; labels [n] uint8 or NULL.  x [N][image_rows][row_pitch] bf16 holding H x W pixels
 *     of C_out channels per image (row_pitch 0 = W C_out rounded up to 8, otherwise a multiple of 8 >= W C_out; image_rows 0 = H,
 *     otherwise >= H).  Pad columns and pad rows of x are never written.  labels_out[j] = labels[i]; both label pointers are NULL
 *     or neither is.
 *   - Which image: position j of the batch is epoch position e = first + j and dataset index i = shuffle ? pi(e) : e.  pi is a
 *     permutation of [0, n) that depends on (seed, epoch, n) alone, not on N, first, the grid or the GPU: a balanced Feistel
 *     network of 6 rounds over 2b bits, b the least with 4^b >= n (4 rounds are measurably biased on domains of a few bits).
 *     With v = (L << b) | R, L and R of b bits, round r = 0..5 maps
 *     (L, R) to (R, L ^ (F_r(R) & (2^b - 1))), F_r(R) = word x of the Philox4x32-10 block at counter (R, 0xC0000000 | r,
 *     epoch lo, epoch hi) with key (seed lo, seed hi).  pi(e) applies the network to e, then again to the result, until the value
 *     is below n (cycle walking: a bijection, with fewer than 4 applications expected since 4^b < 4n; no sort, no scratch).
 *   - Draws: image i's block is Philox4x32-10 at counter (i lo, i hi | 0x80000000, epoch lo, epoch hi) with key (seed lo,
 *     seed hi); oy = umulhi(w.x, 2 pad + 1), ox = umulhi(w.y, 2 pad + 1), flip_i = flip && (w.z >> 31) (probability exactly 1/2).
 *     They depend on the dataset index, not on the batch position: an image gets the same crop in an epoch whatever N or first.
 *     Domains: bit 31 of counter word 1 is set in every counter of this call and bit 30 in the permutation's; word 1 of a dropout
 *     counter (pcnn_dropout_bf16) is the high word of an index below 2^62, so no crop draw or round function coincides with a
 *     dropout draw for any seed, call or epoch, and no round function with a crop draw (i < 2^62).
 *   - Geometry: x[j][h][w][c] = v(c, src[i][h + oy - pad][w' + ox - pad][c]), w' = flip_i ? W - 1 - w : w; a source pixel outside
 *     the image is the byte 0 (so a crop may be all fill).  Channels C <= c < C_out are +0.
 *   - Values: v(c, u) = bf16_rn(RN(RN(RN(float(u) / 255) - mean[c]) / std[c])), ToTensor then Normalize in fp32, each operation an
 *     IEEE round to nearest with no contraction.  The host forms these 256 C values into a table the kernel looks up;
 *     mean_host = NULL means mean 0 and std_host = NULL means std 1, which gives bf16_rn(u / 255).
 * Domain (anything else is PCNN_ERR_ARG with the function and the rule in the message): n, N, H, W >= 1; 0 <= first and first + N
 * <= n; 1 <= C <= 4; C <= C_out <= 8; 0 <= pad <= 64; shuffle and flip 0 or 1; H W C < 2^31 (one image; the dataset is indexed
 * in 64 bits); n H W C < 2^62; row_pitch and image_rows as above; x below 2^62 bytes; mean finite; std finite and > 0; images and
 * x not NULL; x 16-byte aligned; x sharing no byte with images or labels_out, labels_out none with labels or images.
 * Kernel: a CTA of 256 threads per (batch position, block of rows_per_cta output rows), rows_per_cta = ceil(16 KB / (W C_out 2))
 * clamped to 1 .. H; thread 0 runs the generator once for the CTA.  Rows are written as 16-byte vectors of 8 elements when
 * W C_out % 8 == 0, otherwise as single elements, the choice made from the shape.  Stream-ordered; no atomics; the grid depends on
 * the shape alone.
 * pcnn_augment_u8_bf16_info: host only (no GPU, no context), refused as the call refuses.  out8 = { row_pitch, image_rows, b,
 * elements per vector (8 or 1), grid (CTAs), rows_per_cta, row blocks per image, threads per CTA }; lut_out, when not NULL,
 * receives the table, 256 C bf16 bits at [c][u]. */
int pcnn_augment_u8_bf16(pcnn_ctx *ctx, const uint8_t *images_dev, const uint8_t *labels_dev, long long n, int H, int W, int C,
                         long long first, int N, int shuffle, int pad, int flip, unsigned long long seed, unsigned long long epoch,
                         const float *mean_host, const float *std_host, void *x_bf16_dev, int C_out, int row_pitch, int image_rows,
                         uint8_t *labels_out_dev);
int pcnn_augment_u8_bf16_info(long long n, int H, int W, int C, long long first, int N, int shuffle, int pad, int flip, int C_out,
                              int row_pitch, int image_rows, const float *mean_host, const float *std_host, long long *out8,
                              uint16_t *lut_out);
/* Mixed batches (csrc/augment.cu): pcnn_augment_u8_bf16's batch with torchvision's MixUp (mode 1) or CutMix (mode 2) of each
 * image and its partner, as transforms.v2.MixUp / CutMix apply them to the transformed batch.
 *   - Partner: position j's partner is j' = (j + N - 1) mod N (torchvision's roll(1, 0)); N = 1 pairs the image with itself.  Each
 *     image gets its own permutation position, crop and flip exactly as the plain call gives them; a and b below are the fp32
 *     values v(c, u) (before the bf16 rounding) of j's and j''s augmented pixels.
 *   - MixUp: x = bf16_rn(RN(RN(b * RN32(1 - lam)) + RN(a * RN32(lam)))), 1 - lam and lam formed in double and rounded to fp32, no
 *     contraction: what inpt.roll(1, 0).mul_(1.0 - lam).add_(inpt.mul(lam)) computes.  The host forms the fp32 table beside the
 *     bf16 one.
 *   - CutMix: output rows y1 <= h < y2 and columns x1 <= w < x2 (output coordinates, after crop and flip) take the partner's
 *     element, every other pixel j's own: each element has the bits of the plain call's table.
 *   - labels_out[j] = the label of j, labels_b_out[j] = the label of j'.  Channels C <= c < C_out are +0; pad columns and pad rows
 *     of x are never written.
 * Domain: everything pcnn_augment_u8_bf16 requires, with the same messages, plus mode 1 or 2; lam finite with 0 <= lam <= 1;
 * 0 <= x1 <= x2 <= W and 0 <= y1 <= y2 <= H (an empty box is allowed); labels_b_out NULL exactly when labels is; labels_b_out
 * sharing no byte with x, images, labels or labels_out.  The launch is the plain call's (grid, rows per CTA, vector width); lane 0
 * of a second warp walks the partner's permutation and draws its crop beside thread 0's own. */
int pcnn_augment_mix_u8_bf16(pcnn_ctx *ctx, const uint8_t *images_dev, const uint8_t *labels_dev, long long n, int H, int W, int C,
                             long long first, int N, int shuffle, int pad, int flip, unsigned long long seed, unsigned long long epoch,
                             const float *mean_host, const float *std_host, void *x_bf16_dev, int C_out, int row_pitch, int image_rows,
                             uint8_t *labels_out_dev, int mode, double lam, int x1, int y1, int x2, int y2, uint8_t *labels_b_out_dev);
/* Resized batches (csrc/augment.cu): pcnn_augment_u8_bf16's batch at an output size H_out x W_out of its own, with torchvision's
 * RandomResizedCrop((H_out, W_out), scale, ratio, antialias = True) + RandomHorizontalFlip (mode 1, train) or Resize(resize_size) +
 * CenterCrop((H_out, W_out)) (mode 2, eval) on the uint8 image, then the plain call's table v(c, u).  No padding argument.
 *   - Layouts, labels, the permutation pi, the table and channels C <= c < C_out: as pcnn_augment_u8_bf16, with H_out x W_out
 *     pixels per image in x (row_pitch 0 = W_out C_out rounded up to 8, otherwise a multiple of 8 >= W_out C_out; image_rows 0 =
 *     H_out, otherwise >= H_out).  flip_i is the plain call's bit, w.z >> 31 of image i's crop block, so a resized batch flips the
 *     same images as a plain batch of the same (seed, epoch); flip applies in both modes.
 *   - Box (mode 1): torchvision's get_params.  Box block k of image i is Philox4x32-10 at counter (i lo, 0xC0000000 | (8 + k) << 24 |
 *     i hi, epoch lo, epoch hi), key (seed lo, seed hi).  Attempt t = 0..9 takes words (x, y) of block t / 2 for even t, (z, w)
 *     for odd t, as (u_s, u_l); U(u) = RN(RN(RN(float(u >> 8) * 2^-24) * range) + low) in fp32:
 *       s = U(u_s) over (RN32(s0), RN32(RN32(s1) - RN32(s0))), lr = U(u_l) over (L0, RN32(L1 - L0)), L = RN32(log(RN32(r))) on the host;
 *       aspect = double(E(lr)), E the replayable fp32 exponential of the SiLU activations (csrc/pcnn_internal.h exp_f32);
 *       ta = double(H W) * double(s); w = rint(sqrt(ta * aspect)), h = rint(sqrt(ta / aspect)), IEEE double, rint half to even.
 *     The first attempt with 0 < w <= W and 0 < h <= H gives the box, with top = umulhi(b.x, H - h + 1) and left = umulhi(b.y,
 *     W - w + 1) of block 5.  With none: torchvision's central crop (W / H < r0: w = W, h = rint(W / r0); W / H > r1: h = H,
 *     w = rint(H r1); else the image), top = (H - h) / 2, left = (W - w) / 2.  The box is resampled to H_out x W_out.
 *     Domains: word 1 of a box counter is >= 0xC8000000, above every permutation round's (0xC0000000 | r, r < 6); a crop counter has
 *     bit 30 clear (i < 2^62) and a dropout counter bit 31 clear, so no box draw coincides with any of them for any seed or epoch.
 *   - Window (mode 2): the image is resampled to Rh x Rw, the shorter side resize_size and the longer int(resize_size long / short)
 *     (double quotient).  Per axis of resized size R and crop c, the window starts at int(round((R - c) / 2)) (half to even) when
 *     c <= R, else at -((c - R) / 2): positions outside the resized image take the byte 0, as CenterCrop pads.  Only the window's
 *     rows and columns are computed.
 *   - Resample (torch's uint8 bilinear antialias, PIL-SIMD's fixed point): separable, horizontal pass to a uint8 intermediate, then
 *     vertical.  An in -> out axis: scale = in / out, support = max(scale, 1), invscale = scale >= 1 ? 1 / scale : 1, taps =
 *     2 ceil(support) + 1; for output o: centre = scale (o + 0.5), xmin = max(int(centre - support + 0.5), 0), n = clamp(min(int(
 *     centre + support + 0.5), in) - xmin, 0, taps); tap j < n weighs max(0, 1 - |(j + xmin - centre + 0.5) invscale|), then
 *     each is divided by their sum (unless it is 0), all in double with no contraction.  prec = the first p in 0..21 with
 *     int(0.5 + wmax 2^(p+1)) >= 2^15, else 22, wmax the largest weight over every output of the axis (the whole resized axis
 *     in mode 2); weights become int(w 2^prec + 0.5).  Output = clamp((2^(prec-1) + sum_j w_j src[xmin + j]) >> prec, 0, 255) in
 *     int32.  An axis whose size does not change gives its input unchanged.
 *   - x[j][h][w][c] = v(c, u), u the resampled byte at (h, w'), w' = flip_i ? W_out - 1 - w : w.
 * Domain (PCNN_ERR_ARG, in this order, with the function and the rule in the message): ctx, images and x not NULL; labels and
 * labels_out both NULL or neither; n, N, H, W, H_out, W_out >= 1; 0 <= first and first + N <= n; n <= 2^56; 1 <= C <= 4;
 * C <= C_out <= 8; shuffle and flip 0 or 1; mode 1 or 2; H W C < 2^31; n H W C < 2^62; H_out, W_out <= 16384; row_pitch,
 * image_rows and the x size as above; mean finite; std finite and > 0.  Mode 1: s0, s1, r0, r1 each within fp32's normal range
 * [2^-126, 3.4028235e38] (so finite and > 0), s0 <= s1 and r0 <= r1 (torchvision only warns); the central fallback crop not empty.
 * s1 > 1 is allowed: attempts that do not fit fall back.  resize_size is ignored.  Mode 2: 1 <= resize_size <= 16384 and the
 * longer resized side <= 16384; scale and ratio are ignored.  Both: the worst-case box, the whole image resampled to H_out x W_out
 * (mode 1) or Rh x Rw (mode 2), needs at most 33 taps per axis (a downscale of at most 16x); one output row of it fits the dynamic
 * shared memory a launch gets without an opt-in: 48 KB less the kernel's static shared memory (2,224 bytes, out21[20]).  Then x 16-byte aligned, and the plain call's overlap rules.
 * Kernel: a CTA of 256 threads per (batch position, block of rows_per_cta output rows), rows_per_cta the largest <= min(H_out, 32)
 * whose worst-case dynamic shared memory (tap tables of W_out columns and of its rows, and an intermediate of rows_cap source rows x
 * W_out x C bytes) fits that budget.  Thread 0 walks pi and draws the box; the CTA finds both axes' wmax, builds its int16 taps, runs the
 * horizontal pass over the source rows its rows reach and the vertical pass with flip and table, writing 16-byte vectors when
 * W_out C_out % 8 == 0.  Stream-ordered; no atomics; the launch depends on the shape alone.
 * pcnn_augment_resized_u8_bf16_info: host only, refused as the call refuses.  out21 = { row_pitch, image_rows, b, vec, grid,
 * rows_per_cta, row_blocks, threads, dynamic shared bytes, taps_y, taps_x, rows_cap, Rh, Rw, window top, window left, fallback
 * top, left, height, width, static shared bytes } (Rh, Rw = H_out, W_out and the window at 0 in mode 1; the fallback 0 in mode 2); lut_out as the plain
 * info's. */
int pcnn_augment_resized_u8_bf16(pcnn_ctx *ctx, const uint8_t *images_dev, const uint8_t *labels_dev, long long n, int H, int W, int C,
                                 long long first, int N, int shuffle, int flip, unsigned long long seed, unsigned long long epoch,
                                 const float *mean_host, const float *std_host, void *x_bf16_dev, int H_out, int W_out, int C_out,
                                 int row_pitch, int image_rows, uint8_t *labels_out_dev, int mode, double scale_lo, double scale_hi,
                                 double ratio_lo, double ratio_hi, int resize_size);
int pcnn_augment_resized_u8_bf16_info(long long n, int H, int W, int C, long long first, int N, int shuffle, int flip, int H_out,
                                      int W_out, int C_out, int row_pitch, int image_rows, const float *mean_host, const float *std_host,
                                      int mode, double scale_lo, double scale_hi, double ratio_lo, double ratio_hi, int resize_size,
                                      long long *out21, uint16_t *lut_out);
/* TrivialAugmentWide and RandomErasing (csrc/augment.cu): a training batch of torchvision's recipe
 *   (RandomCrop(pad) | RandomResizedCrop) -> RandomHorizontalFlip -> TrivialAugmentWide -> ToTensor -> Normalize -> RandomErasing,
 * in two launches, with the uint8 crop in a caller-owned workspace between them.
 *   - Geometry: resize 0 is pcnn_augment_u8_bf16's crop, pad and flip (an h x w = H x W crop); resize 1 is
 *     pcnn_augment_resized_u8_bf16's mode 1 box, resample and flip (h x w = H_out x W_out; pad must be 0).  Bit for bit those
 *     calls' bytes: the same kernels run at C_out = C with the table v(c, u) = u, into workspace [N][h][ws_pitch] uint16 (the
 *     byte in the low 8 bits; ws_pitch = w C rounded up to 8), at least N h ws_pitch 2 bytes, 16-byte aligned.  Permutation,
 *     labels_out, layouts of x, the table and channels C <= c < C_out: as pcnn_augment_u8_bf16 with H x W replaced by h x w.
 *   - Draws of image i: trivial block k is Philox4x32-10 at counter (i lo, 0xC0000000 | (16 + k) << 24 | i hi, epoch lo, epoch hi),
 *     key (seed lo, seed hi).  Block 0: op = umulhi(x, 14), bin = umulhi(y, 31), sign = z >> 31, erase iff U(w) < RN32(p) with
 *     U(u) = RN(float(u >> 8) 2^-24).  Blocks 1..5: erase attempts t = 0..9 take words (x, y) of block 1 + t / 2 for even t, (z, w)
 *     for odd t, as the resized call's box attempts; block 6 the erase box's (top, left) words.  Domains: word 1 of a trivial
 *     counter is in 0xD0000000 .. 0xD6FFFFFF (i < 2^56): above every box counter (0xC8 .. 0xCD in the top byte) and permutation round
 *     (0xC0), and with bits 31 and 30 set where a crop counter has bit 30 clear and a dropout counter bit 31 clear.
 *   - TrivialAugmentWide (trivial 1: NEAREST, 2: BILINEAR; 0: none, op Identity), num_magnitude_bins 31, fill None, on the uint8
 *     crop [C][h][w], C 1 or 3, as v1 transforms.autoaugment._apply_op on a tensor.  Ops in _augmentation_space's order: 0 Identity,
 *     1 ShearX, 2 ShearY, 3 TranslateX, 4 TranslateY, 5 Rotate, 6 Brightness, 7 Color, 8 Contrast, 9 Sharpness, 10 Posterize,
 *     11 Solarize, 12 AutoContrast, 13 Equalize; sign negates the magnitude of ops 1..9.  Magnitudes: torch.linspace's fp32 values
 *     (0..0.99 for shears and blends, 0..32 for translations, 0..135 for Rotate, 255..0 for Solarize), Posterize 8 - round(bin / 5).
 *     The host forms a table per (op, bin, sign) for this crop size: for ops 1..5, torchvision's _get_inverse_affine_matrix in double
 *     (center (-w/2, -h/2) for shears, translate int(m), Rotate's angle -m), each entry rounded to fp32 then divided in fp32 by
 *     0.5 w (row 0) or 0.5 h (row 1), as _gen_affine_grid rescales theta; ratio = 1 + m and 1 - ratio in double, each rounded to fp32;
 *     Posterize's mask; Solarize's threshold as the least byte >= it.  RN: fp32 round to nearest, no contraction.
 *       blend(a, b) = trunc(clamp(RN(RN(r a) + RN(s b)), 0, 255)); gray = trunc(RN(RN(RN(0.2989 R) + RN(0.587 G)) + RN(0.114 B)));
 *       Brightness blend(u, 0); Color blend(u, gray) (identity at C = 1); Contrast blend(u, mean), mean = RN(S / (h w)), S the exact
 *       sum of gray (C = 3) or of the bytes (C = 1), exact because h w 255 < 2^24; Sharpness (identity when h or w <= 2)
 *       blend(u, b), b = rint(acc) inside the border and u on it, acc the RN sum in row-major tap order of RN(k u) with k = RN32(1 / 13)
 *       and RN32(5 / 13) at the centre; Posterize u & mask; Solarize u >= T ? 255 - u : u; AutoContrast per channel trunc(clamp(RN(
 *       (u - min) scale), 0, 255)), scale = RN(RN(1 / (max - min)) 255) (min 0, scale 1 on a flat channel); Equalize per channel
 *       _scale_channel's integer LUT from the histogram (identity when step = 0).
 *       Geometric ops: output pixel (y, x) takes bx = x + 0.5 - w / 2, by = y + 0.5 - h / 2 (exact), gx = RN(RN(RN(bx v0) +
 *       RN(by v1)) + v2), gy likewise with v3..v5, ix = RN(RN(RN(gx + 1) (0.5 w)) - 0.5), iy likewise; NEAREST takes the byte at
 *       (rint(iy), rint(ix)) (half to even), BILINEAR RN(RN(RN(RN(v_nw RN(s e)) + RN(v_ne RN(s w'))) + RN(v_sw RN(n e))) +
 *       RN(v_se RN(n w'))) with w' = ix - floor(ix), e = 1 - w', n = iy - floor(iy), s = 1 - n, then rint; outside the crop 0.
 *   - Normalise: the table v(c, u) of pcnn_augment_u8_bf16 on the transformed byte.
 *   - RandomErasing(p, (es0, es1), (er0, er1), value = 0) when erase_p > 0: attempt t draws s = U over (RN32(es0), RN32(RN32(es1) -
 *     RN32(es0))) and lr over (L0, RN32(L1 - L0)), L = RN32(log(RN32(r))) as the resized call's box; aspect = double(E(lr));
 *     ea = double(h w) double(s); eh = rint(sqrt(ea aspect)), ew = rint(sqrt(ea / aspect)) in IEEE double.  The first attempt with
 *     eh < h and ew < w gives the box, top = umulhi(x, h - eh + 1), left = umulhi(y, w - ew + 1) of block 6; with none, no erase.
 *     Channels c < C of the box's pixels are bf16 +0.
 * Domain (PCNN_ERR_ARG, in this order): ctx, images, x and the workspace not NULL; labels and labels_out both NULL or neither;
 * resize 0 or 1; trivial 0, 1 or 2; C 1 or 3 when trivial > 0; erase_p finite in [0, 1]; when erase_p > 0, 0 <= es0 <= es1 <= 1 and
 * er0 <= er1 within fp32's normal range; resize 1 with pad 0; then the geometry call's own rules with its messages; then the
 * output layout as pcnn_augment_u8_bf16's at h x w with C_out; h w <= 65536 (256 x 256, so Contrast's sum stays exact); the crop's
 * h w C bytes, rounded up to 16, within the 227 KB of shared memory a CTA may opt into less the kernel's static shared memory
 * (out12[10]): every crop of C <= 3 within 256 x 256 fits, a C = 4 crop (erasing only) up to about 56,800 pixels, so 256 x 256 x 4
 * is refused; x and the workspace 16-byte aligned; workspace_bytes enough; x, labels_out and
 * the workspace sharing no byte with each other, the images or the labels.
 * Kernel: after every check, the geometry call's launch, then one CTA of 512 threads per image (grid min(N, 2^20)) with h w C bytes of dynamic shared
 * memory; shared integer atomics build the histograms (order-free); no other atomics: reruns give the same bits on every H100.
 * pcnn_augment_trivial_u8_bf16_info: host only, refused as the call refuses (bar the pointers).  out12 = { row_pitch, image_rows,
 * h, w, ws_pitch, workspace bytes, vec, grid, threads, dynamic shared bytes, static shared bytes, kernel argument bytes };
 * table_out, when not NULL, receives the table as float [14][31][2][6]; lut_out as the plain info's. */
int pcnn_augment_trivial_u8_bf16(pcnn_ctx *ctx, const uint8_t *images_dev, const uint8_t *labels_dev, long long n, int H, int W, int C,
                                 long long first, int N, int shuffle, int pad, int flip, unsigned long long seed, unsigned long long epoch,
                                 const float *mean_host, const float *std_host, void *x_bf16_dev, int C_out, int row_pitch, int image_rows,
                                 uint8_t *labels_out_dev, int resize, int H_out, int W_out, double scale_lo, double scale_hi,
                                 double ratio_lo, double ratio_hi, int trivial, double erase_p, double erase_scale_lo,
                                 double erase_scale_hi, double erase_ratio_lo, double erase_ratio_hi, void *workspace_dev,
                                 long long workspace_bytes);
int pcnn_augment_trivial_u8_bf16_info(long long n, int H, int W, int C, long long first, int N, int shuffle, int pad, int flip, int resize,
                                      int H_out, int W_out, double scale_lo, double scale_hi, double ratio_lo, double ratio_hi, int trivial,
                                      double erase_p, double erase_scale_lo, double erase_scale_hi, double erase_ratio_lo,
                                      double erase_ratio_hi, int C_out, int row_pitch, int image_rows, const float *mean_host,
                                      const float *std_host, long long *out12, float *table_out, uint16_t *lut_out);
/* Softmax cross-entropy on bf16 logits [N][O], 1 <= O <= 256, labels uint8 [N]:
 *   p = softmax(row) evaluated in double: m = max, den = sum exp(z - m), p_t = exp(z_t - m) / den;
 *   dlogits[n][t] = bf16_rn(float_rn((p_t - [t == label]) * scale)), double -> fp32 -> bf16, each round to nearest even: the
 *     gradient of scale * sum_n CE_n, so scale = 1/N descends the mean loss;
 *   loss[n] = -((z_label - m) - log den) as fp32 (may be NULL);  pred[n] = the first index of the largest logit (may be NULL).
 * A row holding a NaN gets pred -1, a NaN loss and NaN dlogits.  A label >= O gives that row a NaN loss and NaN dlogits (pred is
 * still the argmax).  dlogits == logits (in place) is allowed, any other overlap is not. */
int pcnn_softmax_ce_bf16(pcnn_ctx *ctx, const void *logits_bf16_dev, const uint8_t *labels_dev, int N, int O, float scale,
                         void *dlogits_bf16_dev, float *loss_f32_dev, int *pred_i32_dev);
/* Softmax cross-entropy against a soft target: pcnn_softmax_ce_bf16's layouts, limits, p and pred, with the target row built in
 * fp32 (RN: fp32 round to nearest, no contraction) as torchvision's MixUp / CutMix labels and torch's label smoothing build it:
 *   m_t = RN(RN([t == label_b] RN32(1 - lam)) + RN([t == label] RN32(lam)))   (_mixup_label; labels_b NULL: m_t = [t == label])
 *   q_t = RN(RN(m_t RN32(1 - eps)) + RN32(eps / O))                               (cross_entropy's label_smoothing = eps)
 *   dlogits[n][t] = bf16_rn(float_rn((p_t - q_t) * scale)), p_t in double as the hard call computes it;
 *   loss[n] = fp32 of -sum_t q_t ((z_t - m) - log den) in double, terms with q_t = 0 skipped (may be NULL).
 * Skipping the zero terms differs from torch, whose probability-target path computes 0 * (-Inf) = NaN for a -Inf logit with a
 * zero target; here lam = 1 with eps = 0 gives pcnn_softmax_ce_bf16's bits on every row, whatever labels_b, ±Inf logits included.
 * A row holding a NaN, or a label or label_b >= O, gets a NaN loss and NaN dlogits (pred -1 for NaN, the argmax otherwise).
 * Domain (PCNN_ERR_ARG, one message per rule): lam finite with 0 <= lam <= 1, 0 <= eps <= 1, plus the hard call's; dlogits ==
 * logits (in place) is allowed, any other overlap is not. */
int pcnn_softmax_ce_soft_bf16(pcnn_ctx *ctx, const void *logits_bf16_dev, const uint8_t *labels_dev, const uint8_t *labels_b_dev,
                              double lam, double smoothing, int N, int O, float scale, void *dlogits_bf16_dev, float *loss_f32_dev,
                              int *pred_i32_dev);
/* ------------------------------------------------------------------ dense prediction
 * Transposed convolution (csrc/conv_wide_bwd_tc.cu), as torch.nn.functional.conv_transpose2d(x, w, b, stride, (pad_h, pad_w),
 * (op_h, op_w)) with groups 1 and dilation 1, followed by act (PCNN_ACT_NONE / _SIGMOID / _RELU, the forward epilogues' rule):
 *     H_out = (H - 1) stride - 2 pad_h + R + op_h,   W_out = (W - 1) stride - 2 pad_w + S + op_w
 *     y[n][h][w][co] = act(b[co] + sum_{ci,r,s} x[n][(h + pad_h - r)/stride][(w + pad_w - s)/stride][ci] * f[ci][r][s][co])
 *                      over the (r, s) that divide exactly and give an x pixel inside H x W.
 * It is exactly the input gradient of its adjoint convolution (input H_out x W_out x C_out, K = C_in filters, the same stride and
 * padding, output H x W), pcnn_conv_wide_dgrad_padded(dy = x, filt = f, dx = y), run by a second instantiation of that kernel whose
 * epilogue forms v = fp32 accumulator + b[co] (the accumulator itself with no bias), then act, then one bf16 rounding; the plain
 * input-gradient instantiation is unchanged.  So with no bias and act 0 y is bit for bit pcnn_conv_wide_dgrad_padded, and pixels
 * no window reaches get act(b) (bf16 of +0 with no bias and act 0).
 *   - x is dense bf16 [N][H][W][C_in]; filt_f32_dev the fp32 master [C_in][R][S][C_out] (torch's weight [C_in][C_out][R][S]
 *     permuted (0, 2, 3, 1): the adjoint's KRSC), rounded to bf16 (nearest even) on every call by the input gradient's own
 *     conversion; bias fp32 [C_out] or NULL; y is [N][image_rows][row_pitch] with H_out x W_out pixels of C_out channels
 *     (row_pitch 0 = W_out C_out, image_rows 0 = H_out), the adjoint's x layout.  Pad columns and rows of y are never written.
 *   - Training: the bias / activation gradient is pcnn_conv_bias_act_bwd over y; dx (dense like x) is pcnn_conv_tc_fwd of a wide
 *     plan of the adjoint convolution (no bias, act 0) on dy; dw (fp32 [C_in][R][S][C_out]) is pcnn_conv_wide_wgrad_padded with the
 *     activations swapped, x = dy and dy = x.  The forward and dx read the same bf16 rounding of the master: the forward converts
 *     it on every call, the plan holds what pcnn_conv_plan_set_params or the optimizers made of the same master.
 *   - Domain (PCNN_ERR_ARG, one message per rule naming the called function): N, H, W >= 1; C_in % 8 == 0 and 8 <= C_in <= 256;
 *     C_out % 8 == 0 and C_out >= 8, and C_out <= 256 with a bias or an activation (pcnn_conv_bias_act_bwd); act 0, 1 or 3;
 *     stride 1..4; taps 1..7; 0 <= pad <= taps - 1; 0 <= output_padding < stride; 1 <= H_out, W_out < 2^24; H_out >= stride
 *     when pad_h > 0 (W_out the same); then the adjoint convolution's pitch rules (row_pitch >= W_out C_out and a multiple of 8,
 *     image_rows >= H_out), and at padding (0, 0) the refusal of an adjoint shape the row-Toeplitz plan serves (C_out <= 16 with
 *     few taps), with pcnn_conv_wide_dgrad's messages.  x, y 16-byte aligned.  Reruns are bit-identical.
 * pcnn_conv_transpose_info (host only, no GPU) refuses exactly the same and fills out8 = { H_out, W_out, row_pitch, image_rows,
 * Pt, Qt of the input gradient's pixel block, channel groups, tiles }. */
int pcnn_conv_transpose_info(int N, int H, int W, int C_in, int C_out, int R, int S, int stride, int pad_h, int pad_w, int op_h, int op_w,
                             int row_pitch, int image_rows, int has_bias, int act, int *out8);
int pcnn_conv_transpose_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, const float *filt_f32_dev, const float *bias_f32_dev, void *y_bf16_dev,
                            int N, int H, int W, int C_in, int C_out, int R, int S, int stride, int pad_h, int pad_w, int op_h, int op_w,
                            int row_pitch, int image_rows, int act);
/* Bilinear resizing (csrc/upsample_nhwc.cu), as torch.nn.functional.interpolate(x, size=(H_out, W_out), mode="bilinear",
 * align_corners=False) without antialiasing, up or down, on dense bf16 NHWC maps: x and dx [N][H][W][C], y and dy
 * [N][H_out][W_out][C], any C.  RN is an fp32 operation rounded to nearest, never contracted.  Per axis (in -> out):
 *     scale = RN32(float(in) / float(out));
 *     in == out: i0 = i1 = d, l0 = 1, l1 = 0, decided per axis as torch's CPU kernel decides it (compute_source_index_and_lambda);
 *               torch's CUDA kernel copies only when both axes are unchanged and otherwise takes the general taps, so with one axis
 *               unchanged it reads the neighbour at weight 0 there: a +-Inf neighbour gives NaN on torch's GPU, not here (the
 *               same-index 0 * Inf of a non-finite pixel itself is NaN in both);
 *     otherwise real = RN(RN(scale * RN(d + 0.5)) - 0.5), then real = 0 if real < 0; i0 = min(floor(real), in - 1);
 *               l1 = min(max(RN(real - i0), 0), 1); l0 = RN(1 - l1); i1 = i0 + 1 if i0 < in - 1, else i0.
 * Forward: top = RN(RN(lw0 * x[i0][j0]) + RN(lw1 * x[i0][j1])), bot the same on row i1 (bf16_rn writes every NaN as 0x7FFF),
 *          y[n][h][w][c] = bf16_rn(RN(RN(lh0 * top) + RN(lh1 * bot))).  A 0 weight times +-Inf is NaN, as in torch.
 * Backward, a gather with no atomics: a tap's weight on input index i is l0 if only i0 == i, l1 if only i1 == i and RN(l0 + l1) if
 * both are i; dx[n][i][j][c] = bf16_rn(s), s summed in fp32 from +0 over the output rows h ascending, then the output columns w
 * ascending, whose taps reach (i, j), of RN(RN(wh * ww) * dy[n][h][w][c]).  Reruns give the same bits; torch's CUDA backward adds
 * with atomics, so parity with it is an error bound, not bits.  Every element of y / dx is written, nothing else.
 * Domain (PCNN_ERR_ARG, one message per rule): N, C >= 1; H, W, H_out, W_out 1 .. 16384; each map below 2^62 bytes; x and y
 * 16-byte aligned when C % 8 == 0 (the 8-channel vector path); the two maps must not overlap.
 * pcnn_upsample_bilinear_info (host only) refuses the same and fills out4 = { channels per thread (8 or 1), forward grid,
 * backward grid, threads per CTA }. */
int pcnn_upsample_bilinear_info(int N, int H, int W, int C, int H_out, int W_out, long long *out4);
int pcnn_upsample_bilinear_nhwc_bf16_fwd(pcnn_ctx *ctx, const void *x_bf16_dev, void *y_bf16_dev, int N, int H, int W, int C, int H_out,
                                         int W_out);
int pcnn_upsample_bilinear_nhwc_bf16_bwd(pcnn_ctx *ctx, const void *dy_bf16_dev, void *dx_bf16_dev, int N, int H, int W, int C, int H_out,
                                         int W_out);
/* Per-pixel softmax cross-entropy with an ignore index (csrc/linear_tc.cu), as F.cross_entropy(logits, target,
 * ignore_index=ignore_index) with mean reduction: logits dense bf16 [pixels][O] (1 <= O <= 256), targets uint8 [pixels],
 * ignore_index 0..255 or -1 (none).  Two launches: the first writes count_i32[0] = the number of targets != ignore_index, counted
 * exactly with integer atomics; the second forms scale = fp32(1.0 / double(count)) on the device and runs pcnn_softmax_ce_bf16's
 * kernel with it, so a row whose target is not ignored is bit for bit pcnn_softmax_ce_bf16's row at that scale (a target >= O gives
 * a NaN row, a NaN logit a NaN row and pred -1).  An ignored row gets dlogits +0 and loss 0 whatever its logits; pred is the
 * argmax of every row (-1 for a NaN row).  count 0 makes every row ignored: no NaN dlogits, and the mean loss sum(loss) / count is
 * NaN, as torch's 0 / 0.  loss and pred may be NULL; dlogits == logits (in place) is allowed, no other overlap is.  Domain
 * (PCNN_ERR_ARG): pixels >= 1, 1 <= O <= 256, -1 <= ignore_index <= 255, no NULL context, logits, targets, dlogits or count. */
int pcnn_softmax_ce_pixels_bf16(pcnn_ctx *ctx, const void *logits_bf16_dev, const uint8_t *targets_dev, int pixels, int O, int ignore_index,
                                void *dlogits_bf16_dev, float *loss_f32_dev, int *pred_i32_dev, int *count_i32_dev);
/* Segmentation masks for pcnn_augment_u8_bf16's batch (csrc/augment.cu): masks uint8 [n][H][W] -> masks_out uint8 dense [N][H][W].
 * With the same n, H, W, first, N, shuffle, pad, flip, seed and epoch as the image call, position e = first + j takes mask pi(e)
 * with the crop offsets and flip of the same Philox block the image kernel reads (that kernel is not changed):
 *     masks_out[j][h][w] = masks[pi(e)][h + oy - pad][w' + ox - pad], w' = flip ? W - 1 - w : w,  mask_fill outside the mask,
 * as torchvision's v2.RandomCrop(padding=pad, fill={Mask: mask_fill}) and RandomHorizontalFlip on a tv_tensors.Mask.  shuffle 0,
 * pad 0, flip 0 (an eval batch) copies masks first .. first + N - 1.  Domain: the plain call's rules at C = C_out = 1 with its
 * messages, 0 <= mask_fill <= 255, masks_out disjoint from masks. */
int pcnn_augment_mask_u8(pcnn_ctx *ctx, const uint8_t *masks_dev, long long n, int H, int W, long long first, int N, int shuffle, int pad,
                         int flip, unsigned long long seed, unsigned long long epoch, int mask_fill, uint8_t *masks_out_dev);
/* ------------------------------------------------------------------ image-to-image regression
 * Pixel shuffle and unshuffle (csrc/pixel_shuffle_nhwc.cu), as torch.nn.functional.pixel_shuffle / pixel_unshuffle with upscale /
 * downscale factor r, written for dense bf16 NHWC maps.  With a coarse map [N][H][W][C r^2] and a fine map [N][H r][W r][C]:
 *     fine[n][h r + i][w r + j][c] = coarse[n][h][w][c r^2 + i r + j],   0 <= i, j < r
 * (torch's channel order; TensorFlow's depth_to_space, (i r + j) C + c, is a different permutation).
 *   - pcnn_pixel_shuffle_nhwc_bf16: x is the coarse map [N][H][W][C r^2], y the fine map [N][H r][W r][C];
 *   - pcnn_pixel_unshuffle_nhwc_bf16: x is the fine map [N][H][W][C] with H % r == W % r == 0, y the coarse map
 *     [N][H / r][W / r][C r^2].
 * Each call's own input fixes (N, H, W) and C is the fine map's channel count in both.  The backward of each op is the other op on
 * dy.  Every element of y is a 16-bit copy of one element of x (NaN payloads, +-Inf and -0 unchanged), every element of y is
 * written and nothing else; r = 1 is a copy, as in torch.  Channels per thread: 8 (16-byte accesses) when C % 8 == 0, else 1.
 * Domain (PCNN_ERR_ARG, one message per rule): no NULL context, x or y; N, H, W, C >= 1; 1 <= r <= 8; H and W multiples of r
 * (unshuffle); each map at most 2^31 - 1 elements; x and y 16-byte aligned; x and y disjoint (a permutation cannot run in place).
 * pcnn_pixel_shuffle_info (host only, unshuffle 0 or 1 picks the direction) refuses the same, bar the pointers, and fills
 * out6 = { channels per thread (8 or 1), grid, threads per CTA, shared bytes per CTA, coarse pixels per CTA, fine channels per
 * CTA (C, or a multiple of 8 channels per thread when C r^2 exceeds one CTA's tile) }. */
int pcnn_pixel_shuffle_info(int N, int H, int W, int C, int r, int unshuffle, long long *out6);
int pcnn_pixel_shuffle_nhwc_bf16(pcnn_ctx *ctx, const void *x_bf16_dev, void *y_bf16_dev, int N, int H, int W, int C, int r);
int pcnn_pixel_unshuffle_nhwc_bf16(pcnn_ctx *ctx, const void *x_bf16_dev, void *y_bf16_dev, int N, int H, int W, int C, int r);
/* Regression losses (csrc/regress_loss.cu): F.mse_loss / F.l1_loss of a dense bf16 prediction pred [pixels][C] against the first C
 * channels of a bf16 target [pixels][target_stride] (so a C = 1 prediction compares with channel 0 of a wider map, no copy).
 * RN32 is one fp32 operation rounded to nearest even, never contracted; bf16_rn writes every NaN as 0x7FFF.  Per element:
 *     d = RN32(p - t)
 *     PCNN_LOSS_MSE: term = RN32(d d),  dpred = bf16_rn(RN32(RN32(2 scale) d))
 *     PCNN_LOSS_L1:  term = |d|,        dpred = bf16_rn(RN32(s(d) scale)),  s(d) = +1 (d > 0), -1 (d < 0), +0 (d = +-0 or NaN)
 *     loss[px] = the fp32 sum from +0, in ascending c, of the pixel's terms: unscaled, as pcnn_softmax_ce_bf16's row loss; loss may
 *     be NULL.  The mean loss is sum(loss) / (pixels C), and scale = 1 / (pixels C) makes dpred the gradient of reduction="mean".
 * Special values, as torch's float32 and float64 CPU autograd give them: MSE's dpred is -0 at d = -0, NaN at a NaN d and +-Inf at
 * d = +-Inf (a finite p - t can also overflow to +-Inf in fp32); L1's dpred is +0 at d = +-0 and at a NaN d (torch's sign(NaN) is
 * 0), while its loss term is NaN.  torch's CUDA autograd gives the same classes, with its own roundings (parity within a bf16 ulp).
 * Each element's dpred and each pixel's loss depend on that pixel alone: no cross-CTA reduction, no atomics, and reruns and grids
 * give the same bits.  The 16-byte path (8 channels per thread) runs when C and target_stride are multiples of 8.
 * Domain (PCNN_ERR_ARG, one message per rule): no NULL context, pred, target or dpred; pixels >= 1; 1 <= C <= target_stride; mode
 * PCNN_LOSS_MSE or PCNN_LOSS_L1; scale finite; pred, target, dpred and loss 16-byte aligned; dpred == pred (in place) is allowed,
 * any other overlap of dpred or loss with pred, target or each other is not. */
#define PCNN_LOSS_MSE 0
#define PCNN_LOSS_L1 1
int pcnn_regression_loss_bf16(pcnn_ctx *ctx, const void *pred_bf16_dev, const void *target_bf16_dev, int target_stride, int pixels, int C,
                              int mode, float scale, void *dpred_bf16_dev, float *loss_f32_dev);
/* ------------------------------------------------------------------ variational autoencoders
 * Two more replayable fp32 functions (csrc/pcnn_internal.h), in exp_f32's style: a fixed sequence of round-to-nearest operations
 * with no contraction (RN below), every constant given by its bits, so a numpy float32 replay gives the same bits.
 *   L(e) = log1p_f32(e), log(1 + e) for -1 < e <= 1:
 *     u = RN(1 + e); c = RN(e - RN(u - 1)) (exactly the rounding error of u: both subtractions are exact);
 *     u = 2^k m with m in [sqrt(1/2), sqrt(2)): i = bits(u) + 0x3F800000 - 0x3F3504F3, k = (i >> 23) - 127, m = the float with bits
 *       (i & 0x7FFFFF) + 0x3F3504F3; f = RN(m - 1) (exact);
 *     s = RN(f / RN(2 + f)), z = RN(s s), w = RN(z z); R = RN(RN(z RN(g1 + RN(w g3))) + RN(w RN(g2 + RN(w g4)))), g1 = 0x3F2AAAAA,
 *       g2 = 0x3ECCCCE1, g3 = 0x3E91E9EE, g4 = 0x3E789E26 (fdlibm's logf series in s = f / (2 + f));
 *     hfsq = RN(RN(0.5 f) f); lo = RN(RN(k ln2_lo) + RN(c / u)), ln2_hi = 0x3F317180, ln2_lo = 0x3717F7D1;
 *     L = RN(RN(RN(RN(RN(s RN(hfsq + R)) + lo) - hfsq) + f) + RN(k ln2_hi)).
 *   Its error is at most 0.92 ulp of log1p(e) (measured 0.8684 exhaustively over the 2^24 Box-Muller inputs e = u1 - 1 below, and
 *   0.9154 exhaustively over [2^-30, 1], the largest in [1/4, 1/2); below 2^-30 the result is e within 0.02 ulp).  L(0) = +0.
 *   (sin, cos) = sincos_2pi_f32(k), sin and cos of 2 pi k 2^-24 for integer 0 <= k < 2^24:
 *     octant o = k >> 21, j = k & (2^21 - 1); t = RN(j' 2^-21) with j' = j (o even) or 2^21 - j (o odd): exact, 0 <= t <= 1;
 *     z = RN(t t); S = RN(t P), P = Horner in z of s4 .. s0, each step RN(RN(p z) + s_i), s0 = 0x3F490FDB, s1 = 0xBDA55DE7,
 *       s2 = 0x3B2335DE, s3 = 0xB81965B4, s4 = 0x34A60075; C = Horner in z of c5 .. c0, c0 = 1, c1 = 0xBE9DE9E6, c2 = 0x3C81E0F8,
 *       c3 = 0xB9AAE9DE, c4 = 0x3670F449, c5 = 0xB2D08CC9 (least-squares fits of sin(pi t / 4) / t and cos(pi t / 4) on [0, 1]);
 *     (sin, cos) = o 0: (S, C), 1: (C, S), 2: (C, -S), 3: (S, -C), 4: (-S, -C), 5: (-C, -S), 6: (-C, S), 7: (-S, C).
 *   Each is within 1.72 ulp of the exact value (measured 1.7154 for both over all 2^24 inputs; exact zeros come out as zeros).
 * Gaussian latent (csrc/gaussian_latent.cu): the reparameterization z = mu + exp(lv / 2) eps of a VAE's encoder output, with each
 * row's KL divergence from N(0, I).
 *   - Layout: stats is bf16 [R][ld], mu in columns 0 .. L-1 and the log-variance lv in L .. 2L-1 (a LinearLayer with O = 2L, read in
 *     place; a spatial latent of L channels per pixel is R = N h w rows).  z is bf16 [R][ldz]; kl fp32 [R] or NULL.  Columns 2L ..
 *     ld-1 of stats and L .. ldz-1 of z are never read or written.
 *   - eps[r][j]: element i = r L + j (64-bit) is normal i & 3 of the Philox4x32-10 block at counter (q lo, 0xE0000000 | q hi, call
 *     lo, call hi), q = i >> 2, key (seed lo, seed hi).  A block's words (w0, w1, w2, w3) give normals 0, 1 from the pair (w0, w1) and
 *     2, 3 from (w2, w3) by Box-Muller: u1 = RN(((wa >> 8) + 1) 2^-24) (in (0, 1], exact), rad = sqrt_rn(RN(-2 L(RN(u1 - 1)))),
 *     (sn, cs) = sincos_2pi_f32(wb >> 8); normal 2p = RN(rad cs), 2p + 1 = RN(rad sn).
 *     Domain: word 1 of a latent counter has top byte 0xE0 (q < 2^41 for every allowed shape).  A dropout counter has it below 0x40
 *     (q < 2^62), a crop counter in 0x80 .. 0xBF, a permutation round 0xC0, a box counter 0xC8 .. 0xCD and a trivial-augment counter
 *     0xD0 .. 0xD6, so no latent draw coincides with any other draw of the library for any seed, call or epoch.
 *   - Forward, training 1: z = bf16_rn(RN(mu + RN(E(RN(0.5 lv)) eps))); training 0: z = mu (bit copy, no draw).  mu = lv = 0 gives
 *     z = bf16_rn(eps) (with eps = -0 written as +0), so the same call samples the prior.
 *     kl[r] = RN(0.5 S), S the fp32 sum from +0 in ascending j of RN(RN(RN(RN(mu mu) + E(lv)) - 1) - lv); written in both modes.
 *   - Backward (of a training forward with the same seed and call; nothing is stored, eps is drawn again): with g = float(dz) and
 *     ks = kl_scale (beta / N for a batch mean of beta KL),
 *       dmu = bf16_rn(RN(g + RN(ks mu))),
 *       dlv = bf16_rn(RN(RN(RN(RN(0.5 g) eps) E(RN(0.5 lv))) + RN(RN(ks 0.5) RN(E(lv) - 1))))
 *     into dstats [R][ld] at the columns of mu and lv.
 *   - A row's bits depend only on (seed, call, r, L): no atomics, no dependence on the grid.  16-byte accesses when L, ld and ldz are
 *     multiples of 8, single elements otherwise.
 * Domain (PCNN_ERR_ARG, one message per rule): no NULL context, stats, z (dz, dstats); R >= 1; 1 <= L <= 4096; ld >= 2L; ldz >= L;
 * training 0 or 1; call >= 1 for a training forward and for the backward; kl_scale finite; every pointer 16-byte aligned; z == stats
 * with ldz == ld (in place) or z sharing no byte with stats; kl sharing none with stats or z; dstats == stats (in place) or sharing
 * no byte with it; dstats sharing none with dz.  pcnn_gaussian_latent_info (host only) refuses the shape rules as the calls do and
 * fills out6 = { elements per thread (8 or 1), grid, threads per CTA, shared bytes per CTA, rows per CTA, columns per pass }. */
int pcnn_gaussian_latent_info(int R, int L, int ld, int ldz, long long *out6);
int pcnn_gaussian_latent_bf16_fwd(pcnn_ctx *ctx, const void *stats_bf16_dev, int ld, void *z_bf16_dev, int ldz, float *kl_f32_dev, int R,
                                  int L, unsigned long long seed, unsigned long long call, int training);
int pcnn_gaussian_latent_bf16_bwd(pcnn_ctx *ctx, const void *stats_bf16_dev, int ld, const void *dz_bf16_dev, int ldz, void *dstats_bf16_dev,
                                  int R, int L, unsigned long long seed, unsigned long long call, float kl_scale);
/* Binary cross-entropy with logits (csrc/regress_loss.cu): F.binary_cross_entropy_with_logits of bf16 logits [pixels][C] against
 * the first C channels of bf16 targets [pixels][target_stride], probabilities in [0, 1] (soft targets allowed).  Per element, with
 * x = float(logit), t = float(target), e = E(-|x|):
 *     term = RN(RN((x > 0 ? x : +0) - RN(x t)) + L(e)),
 *     sigma = RN((x >= 0 ? 1 : e) / RN(1 + e)),  dlogits = bf16_rn(RN(scale RN(sigma - t)));
 *     loss[px] = the fp32 sum from +0, in ascending c, of the pixel's terms (unscaled; NULL allowed); scale = 1 / (pixels C) makes
 *     dlogits the gradient of reduction="mean".
 * Special values, against torch's float64 binary_cross_entropy_with_logits and its autograd (sigmoid(x) - t): every finite x gives
 * a finite term and gradient, and |x| > 103.97 gives e = 0, sigma exactly 0 or 1 and the softplus term 0.  A NaN x or t gives NaN
 * in both.  x = +Inf: dlogits = bf16_rn(RN(scale (1 - t))) and x = -Inf: bf16_rn(RN(scale (0 - t))), as torch; the term is NaN at
 * x = +Inf (torch: +Inf for t < 1, NaN at t = 1) and at x = -Inf, t = 0 (torch: NaN), +Inf at x = -Inf, t > 0 (torch: NaN).
 * No cross-CTA reduction and no atomics; the 16-byte path runs when C and target_stride are multiples of 8.
 * Domain (PCNN_ERR_ARG, one message per rule): no NULL context, logits, target or dlogits; pixels >= 1; 1 <= C <= target_stride;
 * scale finite; every pointer 16-byte aligned; dlogits == logits (in place) is allowed, any other overlap of dlogits or loss with
 * logits, target or each other is not. */
int pcnn_bce_logits_bf16(pcnn_ctx *ctx, const void *logits_bf16_dev, const void *target_bf16_dev, int target_stride, int pixels, int C,
                         float scale, void *dlogits_bf16_dev, float *loss_f32_dev);
/* Optimizers for device-trained layers (csrc/optim.cu): one fused update of every parameter tensor of a network per step, as
 * torch.optim.SGD and torch.optim.AdamW (decoupled weight decay) in their single-tensor form, with the bf16 operands of the plans
 * the parameters belong to refreshed in the same pass.
 *   - A table of `count` tensors is validated and uploaded once by pcnn_optim_create; the library allocates the state, zero-filled:
 *     SGD with momentum != 0 has one buffer per tensor (state0 = the momentum buffer b), SGD with momentum 0 none, AdamW two
 *     (state0 = m, state1 = v).  param and grad are fp32 device arrays of n elements; the caller keeps them alive.
 *   - plan_part 1: param is the fp32 master of the plan's filters (KRSC, K R S C elements) or of a linear plan's weights ([O][P][Q][C],
 *     O P Q C elements); 2: the master of its bias (K, or O, elements; the plan must have one); 0: no plan (plan must be NULL),
 *     e.g. batch normalization's gamma and beta.  After the update the plan holds exactly what pcnn_conv_plan_set_params(param) would
 *     give it: wide and linear operands get bf16_rn(p) element by element from the update kernel itself (pad never written), the
 *     bias copy p; a row-Toeplitz plan's filters, where one filter element feeds several operand entries, are gathered afresh from
 *     the updated master by the plan's own kernel, enqueued right after the update (one launch per such plan).
 *   - pcnn_optim_step(ctx, opt, lr): one update kernel over every tensor (CTAs walk fixed chunks of the concatenated tensors; a chunk
 *     table built at creation maps chunk -> tensor), plus the row-Toeplitz gathers.  Stream-ordered, no allocation, no host
 *     synchronisation.  Call it after every backward pass of the step: pcnn_linear_dgrad reads the plan's bf16 weights, which the step
 *     replaces, exactly as the layers' own sgd().  The step count t (kept on the host) is incremented by each call, first call t = 1.
 *     lr < 0 and NaN lr are PCNN_ERR_ARG.
 * Update rules.  Every operation is fp32 round to nearest with no contraction (RN below; a product, then a sum, never an FMA); sqrt
 * and "/" are the correctly rounded IEEE operations.  Element by element, so no result bit depends on the grid or the SM count; NaN
 * and Inf in grads or params propagate by IEEE rules (no clipping, no skipping).  wd is the tensor's weight_decay.
 *   SGD (momentum mu, dampening delta, nesterov):
 *     g' = wd != 0 ? RN(g + RN(wd * p)) : g            (skipped, not multiplied by 0, at wd = 0: 0 * Inf would be NaN)
 *     mu != 0:  b = g' at t = 1 (no dampening on the first step), else b = RN(RN(mu * b) + RN(omega * g')), omega = fp32(1 - delta);
 *               d = nesterov ? RN(g' + RN(mu * b)) : b
 *     mu == 0:  d = g'
 *     p = RN(p + RN((-lr) * d))                          (mu = 0, wd = 0: exactly pcnn_apply_grad_scaled(p, g, n, -lr))
 *   AdamW (beta1, beta2, eps; with the host forming, in double at each step, c2 = fp32(sqrt(1 - beta2^t)) and s = fp32(lr / (1 - beta1^t)),
 *   and per tensor lambda = fp32(1 - double(lr) * double(wd))):
 *     p = RN(p * lambda) when wd != 0
 *     m = RN(m + RN(a1 * RN(g - m))),                    a1 = fp32(1 - beta1)
 *     v = RN(RN(beta2 * v) + RN(RN(a2 * g) * g)),        a2 = fp32(1 - beta2)
 *     den = RN(RN(RN(sqrt(v)) / c2) + eps)
 *     p = RN(p + RN((-s) * RN(m / den)))
 *   AdamW with wd = 0 is Adam.  There is no coupled-L2 Adam, amsgrad, gradient clipping or loss scaling.
 * Vector path: a tensor whose param, grad, state and operand are 16-byte aligned (8-byte for the bf16 operand), with n % 4 == 0 and
 * (with a plan operand) cols % 4 == 0 and pitch % 4 == 0, moves 4 elements per access; any other takes the scalar path.  Both give
 * the same bits.
 * pcnn_optim_create refuses, with PCNN_ERR_ARG and a message naming the rule: NULL ctx, cfg, table or out, count < 1, a NULL param or
 * grad, n <= 0; an unknown kind; momentum < 0, nesterov with momentum <= 0 or dampening != 0, beta1 or beta2 outside [0, 1), eps < 0,
 * weight_decay < 0, any NaN hyperparameter; plan_part outside 0..2, plan_part 0 with a plan or 1..2 without one; plan_part 1 with n
 * other than the plan's master size, plan_part 2 with n != K or for a plan without bias; the same (plan, part) twice; any two of the
 * params, grads and plan operands (bf16 operand rows, bias copy) overlapping.
 * pcnn_optim_state: device pointers of tensor i's state (NULL where the kind keeps none).  pcnn_optim_info: out6 = { tensors,
 * elements, tensors on the vector path, chunks, grid of the update kernel, steps taken }.  pcnn_optim_destroy frees the state and
 * the tables (after the stream's pending work). */
#define PCNN_OPTIM_SGD 0
#define PCNN_OPTIM_ADAMW 1
typedef struct {
    float *param;
    const float *grad;
    long n;
    float weight_decay;
    pcnn_conv_plan *plan;
    int plan_part;          /* 0 none, 1 filters / weights, 2 bias */
} pcnn_optim_tensor;
typedef struct {
    int kind;               /* PCNN_OPTIM_SGD or PCNN_OPTIM_ADAMW */
    float momentum, dampening;
    int nesterov;
    float beta1, beta2, eps;
} pcnn_optim_config;
typedef struct pcnn_optim pcnn_optim;
int pcnn_optim_create(pcnn_ctx *ctx, const pcnn_optim_config *cfg, const pcnn_optim_tensor *tensors, int count, pcnn_optim **out);
int pcnn_optim_step(pcnn_ctx *ctx, pcnn_optim *opt, float lr);
int pcnn_optim_state(pcnn_optim *opt, int i, float **state0_dev, float **state1_dev);
int pcnn_optim_info(pcnn_optim *opt, long *out6);
int pcnn_optim_destroy(pcnn_ctx *ctx, pcnn_optim *opt);

#ifdef __cplusplus
}
#endif
#endif /* PCNN_H_ */
