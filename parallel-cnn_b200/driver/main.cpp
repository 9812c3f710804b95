// parallel-cnn_b200/driver/main.cpp -- the training driver of the reference (Sequential/Main.cpp) on the H100 engine.
//
// Same entry points and the same stdout lines as the reference driver [ref: Sequential/Main.cpp:36-214]:
//   loaddata()      -> reads the four IDX files under data/ (u8 payload kept as u8, return codes checked)
//   learn()         -> "Learning", "error: %e, time_on_cpu: %lf", " Time - %lf"
//   test()          -> "Error Rate: %.2lf%%"
//   forward_pass(), back_pass(), classify(), vectorNorm()
//   the four "Total ... Time" lines
// Two execution modes:
//   default  : the fused path (pcnn_learn / pcnn_test): one kernel per mini-batch step, the whole epoch replayed
//              from CUDA graphs.  --batch 1 (default) replays the reference's per-sample SGD trajectory.
//   --ops    : the reference's own call sequence, operator by operator, through include/layer.h (19 launches per
//              sample; for parity demonstrations, use --limit to bound the run).
// Flags (the reference has none; defaults replay it): --data DIR  --batch B  --epochs E  --limit N  --ops
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <string>
#include <vector>

#include "../../include/layer.h"

double total_convolution_time = 0, total_pooling_time = 0, total_fully_connected_time = 0, total_gradient_time = 0;

struct Dataset {
    uint8_t *images = nullptr;   // [count][784]
    uint8_t *labels = nullptr;
    unsigned count = 0;
};
static Dataset train_set, test_set;
static std::string data_dir = "data";
static int batch = 1, epochs = 1;
static long limit = -1;
static bool ops_mode = false;

// Layers of the network, constructed in the reference's order so rand() hands out the reference's weights
// [ref: Main.cpp:17-20].  In fused mode their parameters are packed into the engine's own vector.
static Layer l_input(0, 0, 28 * 28);
static Layer l_c1(5 * 5, 6, 24 * 24 * 6);
static Layer l_s1(4 * 4, 1, 6 * 6 * 6);
static Layer l_f(6 * 6 * 6, 10, 10);

static void die(int rc, const char *what) {
    if (rc != 0) {
        std::fprintf(stderr, "%s failed (%d): %s\n", what, rc, pcnn_last_error_string());
        std::exit(1);
    }
}

float vectorNorm(float *vec, int n) {   // [ref: Main.cpp:28-34]; vec is a device pointer here
    float host[16];
    l_f.download(host, vec, n);
    float sum = 0.0f;
    for (int i = 0; i < n; ++i) sum += host[i] * host[i];
    return sqrt(sum);
}

static inline void loaddata() {   // [ref: Main.cpp:36-42] -- return codes are checked here
    const std::string d = data_dir + "/";
    int rc = pcnn_mnist_load_u8((d + "train-images.idx3-ubyte").c_str(), (d + "train-labels.idx1-ubyte").c_str(),
                                &train_set.images, &train_set.labels, &train_set.count);
    if (rc) { std::fprintf(stderr, "loaddata: training set: mnist_load code %d\n", rc); std::exit(1); }
    rc = pcnn_mnist_load_u8((d + "t10k-images.idx3-ubyte").c_str(), (d + "t10k-labels.idx1-ubyte").c_str(),
                            &test_set.images, &test_set.labels, &test_set.count);
    if (rc) { std::fprintf(stderr, "loaddata: test set: mnist_load code %d\n", rc); std::exit(1); }
    if (limit > 0 && (unsigned)limit < train_set.count) train_set.count = (unsigned)limit;
}

// ----------------------------------------------------------------------------- operator-by-operator mode
static double forward_pass(const uint8_t *pixels) {   // [ref: Main.cpp:59-105]
    float input[28][28];
    for (int i = 0; i < 28; ++i)
        for (int j = 0; j < 28; ++j) input[i][j] = (float)(pixels[i * 28 + j] / 255.0);   // mnist.h:145 + Main.cpp:64
    l_input.clear(); l_c1.clear(); l_s1.clear(); l_f.clear();
    clock_t t_all = clock(), t0;
    l_input.setOutput((float *)input);
    t0 = clock();
    fp_c1((float(*)[28])l_input.output, (float(*)[24][24])l_c1.preact, (float(*)[5][5])l_c1.weight, l_c1.bias);
    apply_step_function(l_c1.preact, l_c1.output, l_c1.O);
    total_convolution_time += 1000.0 * (clock() - t0) / CLOCKS_PER_SEC;
    t0 = clock();
    fp_s1((float(*)[24][24])l_c1.output, (float(*)[6][6])l_s1.preact, (float(*)[4][4])l_s1.weight, l_s1.bias);
    apply_step_function(l_s1.preact, l_s1.output, l_s1.O);
    total_pooling_time += 1000.0 * (clock() - t0) / CLOCKS_PER_SEC;
    t0 = clock();
    fp_preact_f((float(*)[6][6])l_s1.output, l_f.preact, (float(*)[6][6][6])l_f.weight);
    fp_bias_f(l_f.preact, l_f.bias);
    apply_step_function(l_f.preact, l_f.output, l_f.O);
    total_fully_connected_time += 1000.0 * (clock() - t0) / CLOCKS_PER_SEC;
    return ((double)(clock() - t_all)) / CLOCKS_PER_SEC;
}

static double back_pass() {   // [ref: Main.cpp:107-144]
    clock_t t_all = clock(), t0 = clock();
    bp_weight_f((float(*)[6][6][6])l_f.d_weight, l_f.d_preact, (float(*)[6][6])l_s1.output);
    bp_bias_f(l_f.bias, l_f.d_preact);
    total_fully_connected_time += 1000.0 * (clock() - t0) / CLOCKS_PER_SEC;
    t0 = clock();
    bp_output_s1((float(*)[6][6])l_s1.d_output, (float(*)[6][6][6])l_f.weight, l_f.d_preact);
    bp_preact_s1((float(*)[6][6])l_s1.d_preact, (float(*)[6][6])l_s1.d_output, (float(*)[6][6])l_s1.preact);
    bp_weight_s1((float(*)[4][4])l_s1.d_weight, (float(*)[6][6])l_s1.d_preact, (float(*)[24][24])l_c1.output);
    bp_bias_s1(l_s1.bias, (float(*)[6][6])l_s1.d_preact);
    total_pooling_time += 1000.0 * (clock() - t0) / CLOCKS_PER_SEC;
    t0 = clock();
    bp_output_c1((float(*)[24][24])l_c1.d_output, (float(*)[4][4])l_s1.weight, (float(*)[6][6])l_s1.d_preact);
    bp_preact_c1((float(*)[24][24])l_c1.d_preact, (float(*)[24][24])l_c1.d_output, (float(*)[24][24])l_c1.preact);
    bp_weight_c1((float(*)[5][5])l_c1.d_weight, (float(*)[24][24])l_c1.d_preact, (float(*)[28])l_input.output);
    bp_bias_c1(l_c1.bias, (float(*)[24][24])l_c1.d_preact);
    total_convolution_time += 1000.0 * (clock() - t0) / CLOCKS_PER_SEC;
    t0 = clock();
    apply_grad(l_f.weight, l_f.d_weight, l_f.M * l_f.N);
    apply_grad(l_s1.weight, l_s1.d_weight, l_s1.M * l_s1.N);
    apply_grad(l_c1.weight, l_c1.d_weight, l_c1.M * l_c1.N);
    total_gradient_time += 1000.0 * (clock() - t0) / CLOCKS_PER_SEC;
    return ((double)(clock() - t_all)) / CLOCKS_PER_SEC;
}

static unsigned int classify(const uint8_t *pixels) {   // [ref: Main.cpp:186-200]
    float res[10];
    forward_pass(pixels);
    l_f.download(res, l_f.output, 10);
    unsigned int best = 0;
    for (int i = 1; i < 10; ++i)
        if (res[best] < res[i]) best = i;
    return best;
}

// ----------------------------------------------------------------------------- fused mode plumbing
static void pack_params_into_engine() {
    float p[PCNN_NPARAM];
    l_c1.download(p + PCNN_OFF_C1W, l_c1.weight, 150);  l_c1.download(p + PCNN_OFF_C1B, l_c1.bias, 6);
    l_s1.download(p + PCNN_OFF_S1W, l_s1.weight, 16);   l_s1.download(p + PCNN_OFF_S1B, l_s1.bias, 1);
    l_f.download(p + PCNN_OFF_FW, l_f.weight, 2160);    l_f.download(p + PCNN_OFF_FB, l_f.bias, 10);
    die(pcnn_set_params(pcnn_dropin::ctx(), p), "pcnn_set_params");
}

static void learn() {   // [ref: Main.cpp:146-184]
    float err = 0.0f;
    int iter = epochs;
    double time_taken = 0.0;
    std::fprintf(stdout, "Learning\n");
    pcnn_ctx *c = pcnn_dropin::ctx();
    while (iter-- > 0) {
        auto t0 = std::chrono::steady_clock::now();
        if (ops_mode) {
            err = 0.0f;
            for (unsigned i = 0; i < train_set.count; ++i) {
                forward_pass(train_set.images + (size_t)i * 784);
                l_f.bp_clear(); l_s1.bp_clear(); l_c1.bp_clear();
                makeError(l_f.d_preact, l_f.output, train_set.labels[i], 10);
                err += vectorNorm(l_f.d_preact, 10);
                back_pass();
            }
            err /= train_set.count;
        } else {
            die(pcnn_learn(c, batch, 1, &err), "pcnn_learn");
        }
        time_taken += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        std::fprintf(stdout, "error: %e, time_on_cpu: %lf\n", err, time_taken);
        if (err < threshold) {
            std::fprintf(stdout, "Training complete, error less than threshold\n\n");
            break;
        }
    }
    std::fprintf(stdout, "\n Time - %lf\n", time_taken);
}

static void test() {   // [ref: Main.cpp:202-214]
    long error = 0;
    if (ops_mode) {
        for (unsigned i = 0; i < test_set.count; ++i)
            if (classify(test_set.images + (size_t)i * 784) != test_set.labels[i]) ++error;
    } else {
        die(pcnn_test(pcnn_dropin::ctx(), &error), "pcnn_test");
    }
    std::fprintf(stdout, "Error Rate: %.2lf%%\n", double(error) / double(test_set.count) * 100.0);
}

int main(int argc, const char **argv) {
    for (int i = 1; i < argc; ++i) {
        std::string a = argv[i];
        auto next = [&]() -> const char * { if (i + 1 >= argc) { std::fprintf(stderr, "missing value for %s\n", a.c_str()); std::exit(2); } return argv[++i]; };
        if (a == "--data") data_dir = next();
        else if (a == "--batch") batch = std::atoi(next());
        else if (a == "--epochs") epochs = std::atoi(next());
        else if (a == "--limit") limit = std::atol(next());
        else if (a == "--ops") ops_mode = true;
        else { std::fprintf(stderr, "usage: %s [--data DIR] [--batch B] [--epochs E] [--limit N] [--ops]\n", argv[0]); return 2; }
    }
    srand(time(NULL));   // as the reference does: too late to affect the statically constructed weights [ref: Main.cpp:46]
    loaddata();
    if (!ops_mode) {
        pcnn_ctx *c = pcnn_dropin::ctx();
        pack_params_into_engine();
        die(pcnn_dataset_upload(c, PCNN_TRAIN_SET, train_set.images, PCNN_U8, train_set.labels, train_set.count), "pcnn_dataset_upload(train)");
        die(pcnn_dataset_upload(c, PCNN_TEST_SET, test_set.images, PCNN_U8, test_set.labels, test_set.count), "pcnn_dataset_upload(test)");
    } else if (limit > 0 && (unsigned)limit < test_set.count) {
        test_set.count = (unsigned)limit;
    }
    learn();
    test();
    std::printf("Total Convolution Time: %f ms\n", total_convolution_time);
    std::printf("Total Pooling Time: %f ms\n", total_pooling_time);
    std::printf("Total Fully Connected Time: %f ms\n", total_fully_connected_time);
    std::printf("Total Time on applying gradients: %f ms\n", total_gradient_time);
    return 0;
}
