// oracle/ref_cuda_harness.cu -- TEST / BASELINE INFRASTRUCTURE ONLY (never linked into the product).
//
// Times the reference's OWN GPU path (CUDA/main.cu + CUDA/layer.cu, unmodified, compiled where they lie under
// the reference sources for sm_90a) on the same H100 as the engine: the only GPU-vs-GPU anchor this project has
// (BASELINE.md section 3.4, SURVEY.md 2.2).  The reference's own timer wraps asynchronous launches with clock() and never
// synchronises (CUDA/main.cu:71-72, 107-108, 115-117, 160-161), so this harness brackets learn() with
// cudaDeviceSynchronize() and a wall clock instead.  main.cu is included as a translation unit with its main() renamed,
// exactly like ref_harness.cpp does for Sequential/Main.cpp; no reference text is copied.
//
// NOT an oracle: two of its kernels are numerically wrong (SURVEY.md 2.2: bp_bias_s1, bp_output_c1) and it uses expf.
//
//   usage: cuda_ref_bench [samples]     (cwd must contain data/, as the reference requires; default 20000 samples)
#include <chrono>
#include <cstdio>
#include <cstdlib>

#define main ref_cuda_main
#include "main.cu"   // -I/root/reference/CUDA
#undef main

int main(int argc, char **argv) {
    const unsigned want = argc > 1 ? (unsigned)atoi(argv[1]) : 20000u;
    if (cuInit(0) != CUDA_SUCCESS) {
        fprintf(stderr, "cuInit failed\n");
        return 1;
    }
    loaddata();                                       // CUDA/main.cu:33-39
    if (train_cnt == 0) {
        fprintf(stderr, "no training data (cwd must contain data/)\n");
        return 2;
    }
    if (want < train_cnt) train_cnt = want;           // bounded sample of the same loop
    // warm-up: first launches pay module load + cuBLAS initialisation
    const unsigned full = train_cnt;
    train_cnt = full < 256 ? full : 256;
    learn();
    cudaDeviceSynchronize();
    train_cnt = full;
    const auto t0 = std::chrono::steady_clock::now();
    learn();                                          // CUDA/main.cu:165-208: one epoch over train_cnt samples, batch 1
    cudaDeviceSynchronize();
    const double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    printf("REF_CUDA samples=%u seconds=%.6f images_per_s=%.1f\n", train_cnt, s, train_cnt / s);
    return 0;
}
