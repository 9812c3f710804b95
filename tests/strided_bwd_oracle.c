/* tests/strided_bwd_oracle.c -- direct-loop restatement of the backward passes of the strided NHWC convolution (TEST
 * INFRASTRUCTURE ONLY).  The same conventions as orc_conv_wgrad_nhwc / orc_conv_dgrad_nhwc in oracle/lenet_oracle.c (KRSC
 * filters, NHWC activations, double accumulation), with the window step `stride` of orc_conv_fwd_nhwc_strided:
 * dy [N][(H-R)/stride+1][(W-S)/stride+1][K].  tests/test_conv_strided_cpu.py compiles it with the oracle's parity flags
 * (no FMA contraction) and pins the float64 references of tests/conv_ref_strided.py to it. */

/* dw[k][r][s][c] = sum_{n,p,q} dy[n][p][q][k] * x[n][p*stride+r][q*stride+s][c] */
void orc_conv_wgrad_nhwc_strided(const float *x, const float *dy, float *dw,
                                 int N, int H, int W, int C, int K, int R, int S, int stride) {
    int P = (H - R) / stride + 1, Q = (W - S) / stride + 1;
    for (int k = 0; k < K; ++k)
        for (int r = 0; r < R; ++r)
            for (int s = 0; s < S; ++s)
                for (int c = 0; c < C; ++c) {
                    double acc = 0.0;
                    for (int n = 0; n < N; ++n)
                        for (int p = 0; p < P; ++p)
                            for (int q = 0; q < Q; ++q)
                                acc += (double)dy[(((long)n * P + p) * Q + q) * K + k] *
                                       (double)x[(((long)n * H + p * stride + r) * W + q * stride + s) * C + c];
                    dw[((k * R + r) * S + s) * C + c] = (float)acc;
                }
}

/* dx[n][h][w][c] = sum_{k,r,s} dy[n][(h-r)/stride][(w-s)/stride][k] * w[k][r][s][c] over the (r, s) with stride | h-r,
 * stride | w-s and the dy pixel inside [P x Q]; 0 where no window covers (h, w) */
void orc_conv_dgrad_nhwc_strided(const float *dy, const float *w, float *dx,
                                 int N, int H, int W, int C, int K, int R, int S, int stride) {
    int P = (H - R) / stride + 1, Q = (W - S) / stride + 1;
    for (int n = 0; n < N; ++n)
        for (int h = 0; h < H; ++h)
            for (int ww = 0; ww < W; ++ww)
                for (int c = 0; c < C; ++c) {
                    double acc = 0.0;
                    for (int r = 0; r < R; ++r) {
                        int ph = h - r;
                        if (ph < 0 || ph % stride) continue;
                        int p = ph / stride;
                        if (p >= P) continue;
                        for (int s = 0; s < S; ++s) {
                            int qw = ww - s;
                            if (qw < 0 || qw % stride) continue;
                            int q = qw / stride;
                            if (q >= Q) continue;
                            for (int k = 0; k < K; ++k)
                                acc += (double)dy[(((long)n * P + p) * Q + q) * K + k] *
                                       (double)w[((k * R + r) * S + s) * C + c];
                        }
                    }
                    dx[(((long)n * H + h) * W + ww) * C + c] = (float)acc;
                }
}
