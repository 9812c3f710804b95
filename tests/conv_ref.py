"""float64 references of the NHWC convolution passes, and the tiling regime a shape puts the tensor-core kernels in (TEST
INFRASTRUCTURE ONLY).

The C oracle (orc_conv_*_nhwc in oracle/lenet_oracle.c) is a single-threaded direct loop: about 11 G multiply-adds per pass at
BASELINE config 5 with N = 128.  The references here compute the same sums in float64 as im2col-by-shift + one BLAS matmul,
a few images at a time (CHUNK), so host memory stays near a few hundred MB whatever N is.  Operands may be of any numeric dtype
(uint8 / int8 integers, float32 bf16-rounded values); they are converted to float64 chunk by chunk.
tests/test_oracle_cpu.py pins them to the C oracle.
"""
import numpy as np

CHUNK = 8          # images per evaluation step


def _cols(x, R, S, stride, P, Q):
    """x [n, H, W, C] -> float64 [n * P * Q, R * S * C]: row (n, p, q) holds the window of output pixel (p, q)"""
    n, C = x.shape[0], x.shape[3]
    out = np.empty((n, P, Q, R, S, C))
    for r in range(R):
        for s in range(S):
            out[:, :, :, r, s, :] = x[:, r:r + (P - 1) * stride + 1:stride, s:s + (Q - 1) * stride + 1:stride, :]
    return out.reshape(n * P * Q, R * S * C)


def conv_fwd_f64(x, f, bias=None, stride=1):
    """y[n][p][q][k] = bias[k] + sum_{r,s,c} x[n][p*stride + r][q*stride + s][c] * f[k][r][s][c]; float64 [N, P, Q, K]"""
    N, H, W, _ = x.shape
    K, R, S, _ = f.shape
    P, Q = (H - R) // stride + 1, (W - S) // stride + 1
    fm = np.asarray(f, np.float64).reshape(K, -1).T
    y = np.empty((N, P, Q, K))
    for n0 in range(0, N, CHUNK):
        n1 = min(N, n0 + CHUNK)
        y[n0:n1] = (_cols(x[n0:n1], R, S, stride, P, Q) @ fm).reshape(n1 - n0, P, Q, K)
    if bias is not None:
        y += np.asarray(bias, np.float64)
    return y


def conv_wgrad_f64(x, dy, R, S):
    """dw[k][r][s][c] = sum_{n,p,q} dy[n][p][q][k] * x[n][p + r][q + s][c] (stride 1); float64 [K, R, S, C]"""
    N, _, _, C = x.shape
    _, P, Q, K = dy.shape
    dw = np.zeros((K, R * S * C))
    for n0 in range(0, N, CHUNK):
        n1 = min(N, n0 + CHUNK)
        dw += np.asarray(dy[n0:n1], np.float64).reshape(-1, K).T @ _cols(x[n0:n1], R, S, 1, P, Q)
    return dw.reshape(K, R, S, C)


def conv_dgrad_f64(dy, f):
    """dx[n][h][w][c] = sum_{k,r,s} dy[n][h - r][w - s][k] * f[k][r][s][c] (stride 1, valid); float64 [N, P+R-1, Q+S-1, C]"""
    N, P, Q, K = dy.shape
    _, R, S, C = f.shape
    fm = np.asarray(f, np.float64).reshape(K, -1)
    dx = np.zeros((N, P + R - 1, Q + S - 1, C))
    for n0 in range(0, N, CHUNK):
        n1 = min(N, n0 + CHUNK)
        d = (np.asarray(dy[n0:n1], np.float64).reshape(-1, K) @ fm).reshape(n1 - n0, P, Q, R, S, C)
        for r in range(R):
            for s in range(S):
                dx[n0:n1, r:r + P, s:s + Q, :] += d[:, :, :, r, s, :]
    return dx


# --------------------------------------------------------------------------- tiling regimes (host-side plan queries only)
# The three kernels are persistent: min(work items, SMs) CTAs loop over tiles (forward, weight gradient) or over a share of
# the rows of a column strip (input gradient), fed through a ring of `stages` shared-memory stages.  These say how far a
# shape drives those loops on a GPU with `sm_count` SMs.

def fwd_regime(pkg, N, H, W, C, K, R, S, sm_count, stride=1, row_pitch=None, image_rows=0):
    pl = pkg.conv_tc_plan_info(N, H, W, C, K, R, S, stride, row_pitch, image_rows)
    grid = min(pl["tiles"], sm_count)
    return dict(pl, grid=grid, min_tiles_per_cta=pl["tiles"] // grid)


def wgrad_regime(pkg, N, H, W, C, K, R, S, sm_count):
    b = pkg.conv_bwd_plan_info(N, H, W, C, K, R, S)
    if not b["wgrad_tc"]:
        return None
    P, Q, RB, PC = H - R + 1, W - S + 1, b["wgrad_rb"], b["wgrad_pc"]
    n_pb, n_ch = -(-P // RB), -(-Q // PC)
    tiles = N * n_pb * n_ch
    grid = min(tiles, sm_count)
    return dict(stages=b["wgrad_stages"], RB=RB, PC=PC, n_pb=n_pb, n_ch=n_ch, tiles=tiles, grid=grid,
                min_tiles_per_cta=tiles // grid, max_tiles_per_cta=-(-tiles // grid), ragged=P % RB != 0)


def dgrad_regime(pkg, N, H, W, C, K, R, S, sm_count):
    b = pkg.conv_bwd_plan_info(N, H, W, C, K, R, S)
    if not b["dgrad_tc"]:
        return None
    T, nstrips = N * H, b["dgrad_strips"]
    grid = min(T * nstrips, sm_count)
    rows, crossing = [], 0
    for strip in range(nstrips):                      # the split of conv_dgrad_tc.cu (RowWalk)
        cnt = -(-(grid - strip) // nstrips)
        L = -(-T // cnt)
        for idx in range(cnt):
            t0, t1 = min(idx * L, T), min(idx * L + L, T)
            if t1 > t0:
                rows.append(t1 - t0)
                crossing += t0 // H != (t1 - 1) // H
    return dict(stages=b["dgrad_stages"], grid=grid, max_rows_per_share=max(rows), min_rows_per_share=min(rows),
                shares_crossing_images=crossing)


# --------------------------------------------------------------------------- the multi-tile cases of tests/test_conv_tc_gpu.py
SM_COUNTS = (114, 132)       # H100 PCIe / SXM: the cases below reach their regime on both (test_host_cpu.py)

FWD_MULTI = [  # N, H, W, C, K, R, S, stride, row_pitch, image_rows, bias
    (128, 224, 224, 3, 64, 3, 3, 1, 672, 0, True),      # BASELINE config 5 as bench.py runs it: 12,544 tiles, V = 2 alignment variants
    (64, 224, 224, 3, 64, 3, 3, 2, 672, 0, True),       # stride 2: 1,568 tiles
    (8192, 28, 28, 1, 6, 5, 5, 1, 32, 32, True),        # LeNet c1, [N][32][32] layout with bias: 2,048 tiles
]
BWD_MULTI = [  # N, H, W, C, K, R, S, row_pitch, image_rows
    (128, 224, 224, 3, 64, 3, 3, 0, 0),                 # BASELINE config 5 as bench.py runs it
    (1024, 28, 28, 1, 6, 5, 5, 32, 32),                 # LeNet c1: K = 6 -> 64 through the padded dy copy; [N][32][32] layout
    (96, 40, 72, 3, 96, 3, 3, 0, 0),                    # K = 96: dy read in place (dy_channels), boxes zero-filled to 128
    (128, 40, 40, 1, 128, 3, 3, 0, 0),                  # K = 128: two 64-filter groups
    (96, 24, 40, 2, 256, 3, 3, 88, 26),                 # K = 256, C = 2; strided layout (pitch 88 > 80, 26 rows per image)
    (7, 337, 136, 2, 64, 3, 3, 0, 0),                   # C = 2: ragged last row block (335 = 83 x 4 + 3), three pixel chunks
    (246, 15, 24, 4, 64, 3, 3, 0, 0),                   # C = 4: ragged last row block (13 = 6 x 2 + 1)
    (64, 21, 40, 8, 64, 3, 3, 0, 0),                    # C = 8: input gradient only
    (246, 17, 24, 1, 64, 5, 5, 0, 0),                   # 5x5, C = 1: ragged last row block
    (64, 21, 40, 3, 64, 5, 5, 0, 0),                    # 5x5, C = 3: input gradient only
    (120, 40, 72, 1, 64, 7, 7, 0, 0),                   # 7x7, C = 1
    (3, 151, 542, 1, 64, 3, 3, 544, 0),                 # C = 1: 17 pixel chunks, ragged last row block, W*C % 8 != 0 (guarded copies)
]
WGRAD_PAD = [  # N, H, W, C, K, R, S, row_pitch, image_rows: weight gradient with NaN row padding
    (3, 151, 542, 1, 64, 3, 3, 552, 160),               # guard (W*C*2 % 16 != 0), 17 pixel chunks, ragged last row block
    (1024, 28, 28, 1, 6, 5, 5, 32, 32),                 # guard, LeNet c1 at pitch 32
    (7, 337, 136, 2, 64, 3, 3, 288, 340),               # no guard (W*C*2 % 16 == 0), pitch > W*C; three chunks, ragged
]
