"""float64 references of the backward passes of the strided NHWC convolution, the tiling regime a strided shape puts the
backward tensor-core kernels in, and the multi-tile strided cases (TEST INFRASTRUCTURE ONLY).

The same method as tests/conv_ref.py (im2col-by-shift + one BLAS matmul, CHUNK images at a time), with the window step
`stride` of conv_ref.conv_fwd_f64.  At stride 1 every function here computes what its conv_ref counterpart computes.
tests/test_conv_strided_cpu.py pins them to the direct loops of tests/strided_bwd_oracle.c.
"""
import numpy as np

import conv_ref as CR


def out_size(H, W, R, S, stride):
    return (H - R) // stride + 1, (W - S) // stride + 1


def conv_wgrad_f64(x, dy, R, S, stride=1):
    """dw[k][r][s][c] = sum_{n,p,q} dy[n][p][q][k] * x[n][p*stride + r][q*stride + s][c]; float64 [K, R, S, C]"""
    N, _, _, C = x.shape
    _, P, Q, K = dy.shape
    dw = np.zeros((K, R * S * C))
    for n0 in range(0, N, CR.CHUNK):
        n1 = min(N, n0 + CR.CHUNK)
        dw += np.asarray(dy[n0:n1], np.float64).reshape(-1, K).T @ CR._cols(x[n0:n1], R, S, stride, P, Q)
    return dw.reshape(K, R, S, C)


def conv_dgrad_f64(dy, f, H, W, stride=1):
    """dx[n][h][w][c] = sum_{k,r,s} dy[n][(h - r)/stride][(w - s)/stride][k] * f[k][r][s][c] over the (r, s) that divide
    exactly; float64 [N, H, W, C].  H and W are needed: at stride > 1 several image sizes give the same dy."""
    N, P, Q, K = dy.shape
    _, R, S, C = f.shape
    assert out_size(H, W, R, S, stride) == (P, Q)
    fm = np.asarray(f, np.float64).reshape(K, -1)
    dx = np.zeros((N, H, W, C))
    for n0 in range(0, N, CR.CHUNK):
        n1 = min(N, n0 + CR.CHUNK)
        d = (np.asarray(dy[n0:n1], np.float64).reshape(-1, K) @ fm).reshape(n1 - n0, P, Q, R, S, C)
        for r in range(R):
            for s in range(S):
                dx[n0:n1, r:r + (P - 1) * stride + 1:stride, s:s + (Q - 1) * stride + 1:stride, :] += d[:, :, :, r, s, :]
    return dx


def wgrad_regime(pkg, N, H, W, C, K, R, S, sm_count, stride=1):
    b = pkg.conv_bwd_plan_info(N, H, W, C, K, R, S, stride)
    if not b["wgrad_tc"]:
        return None
    (P, Q), RB, PC = out_size(H, W, R, S, stride), b["wgrad_rb"], b["wgrad_pc"]
    n_pb, n_ch = -(-P // RB), -(-Q // PC)
    tiles = N * n_pb * n_ch
    grid = min(tiles, sm_count)
    return dict(stages=b["wgrad_stages"], RB=RB, PC=PC, n_pb=n_pb, n_ch=n_ch, tiles=tiles, grid=grid,
                min_tiles_per_cta=tiles // grid, max_tiles_per_cta=-(-tiles // grid), ragged=P % RB != 0)


def dgrad_regime(pkg, N, H, W, C, K, R, S, sm_count, stride=1):
    """the split of conv_dgrad_tc.cu (RowWalk) over N * ceil(H / stride) units of `stride` dx rows"""
    b = pkg.conv_bwd_plan_info(N, H, W, C, K, R, S, stride)
    if not b["dgrad_tc"]:
        return None
    U = -(-H // stride)
    T, nstrips = N * U, b["dgrad_strips"]
    grid = min(T * nstrips, sm_count)
    units, crossing = [], 0
    for strip in range(nstrips):
        cnt = -(-(grid - strip) // nstrips)
        L = -(-T // cnt)
        for idx in range(cnt):
            t0, t1 = min(idx * L, T), min(idx * L + L, T)
            if t1 > t0:
                units.append(t1 - t0)
                crossing += t0 // U != (t1 - 1) // U
    return dict(stages=b["dgrad_stages"], ring=b["dgrad_ring"], grid=grid, max_units_per_share=max(units),
                min_units_per_share=min(units), shares_crossing_images=crossing)


# Cases sized like conv_ref.BWD_MULTI: on 114 and 132 SMs every weight-gradient CTA runs more than 2 x stages tiles and the
# input-gradient shares are longer than the stage ring and cross images (tests/test_conv_strided_cpu.py checks that).
BWD_STRIDED_MULTI = [  # N, H, W, C, K, R, S, stride, row_pitch, image_rows
    (128, 224, 224, 3, 64, 3, 3, 2, 0, 0),              # BASELINE config 5 at stride 2: 111 x 111 dy pixels
    (1024, 28, 28, 1, 6, 5, 5, 2, 32, 32),              # LeNet c1 at stride 2: K = 6 -> 64 through the padded dy copy; [N][32][32]
    (256, 40, 72, 2, 64, 3, 3, 3, 0, 42),               # C = 2, stride 3: rows per image padded to a multiple of 3
    (512, 64, 100, 1, 64, 3, 3, 4, 104, 0),             # stride 4 > R: uncovered rows and columns between windows; guarded copies
    (96, 40, 72, 3, 32, 3, 3, 2, 0, 0),                 # K = 32: dy read in place, boxes zero-filled to 64
    (160, 40, 40, 1, 128, 3, 3, 2, 0, 0),               # K = 128: two 64-filter groups
    (4, 4006, 40, 1, 64, 3, 3, 2, 0, 0),                # ragged last row block (2,002 dy rows = 500 x 4 + 2)
    (256, 42, 72, 4, 64, 3, 3, 2, 0, 0),                # (H-R) % 2 != 0 and (W-S) % 2 != 0: last row and column uncovered
    (120, 40, 72, 1, 64, 7, 7, 2, 0, 0),                # 7x7 at stride 2
    (256, 21, 40, 8, 64, 3, 3, 2, 0, 0),                # C = 8: no weight-gradient plan, input gradient only
    (256, 21, 40, 3, 64, 5, 5, 2, 0, 0),                # 5x5, C = 3: no weight-gradient plan, input gradient only
]
