"""The NHWC max pool on the device (pcnn_maxpool_nhwc_bf16_fwd / _bwd, MaxPoolLayer): y, argmax and dx bit-identical to the numpy
reference of tests/maxpool_ref.py (pinned to torch's CPU max pool by test_maxpool_nhwc_cpu.py) in every layout and window shape,
torch's CUDA max pool on the same channels-last bf16 tensors, every refusal, and a conv -> pool -> conv -> pool stack trained on
MNIST digits."""
import numpy as np
import pytest
import torch

import conv_ref_strided as CS
import maxpool_ref as MR

pytestmark = pytest.mark.gpu

NAN_BF16 = 0x7FC0
LR = 2.0 ** -20

CASES = [  # id, N, H, W, C, R, S, stride, pad_h, pad_w, row_pitch (0 = Q*C rounded up to 8), image_rows (0 = P)
    ("lenet-24x24x6-2x2s2-pitched", 16, 24, 24, 6, 2, 2, 2, 0, 0, 80, 14),
    ("c1-2x2s2", 2, 10, 9, 1, 2, 2, 2, 0, 0, 0, 0),
    ("c3-2x2s2", 2, 10, 9, 3, 2, 2, 2, 0, 0, 0, 0),
    ("c16-2x2s2", 2, 10, 9, 16, 2, 2, 2, 0, 0, 0, 0),
    ("c24-2x2s2", 2, 10, 9, 24, 2, 2, 2, 0, 0, 0, 0),
    ("c64-2x2s2", 2, 10, 9, 64, 2, 2, 2, 0, 0, 0, 0),
    ("c256-2x2s2", 2, 10, 9, 256, 2, 2, 2, 0, 0, 0, 0),
    ("c320-3x3s2p1", 2, 9, 7, 320, 3, 3, 2, 1, 1, 0, 0),
    ("3x3s2p1-odd", 2, 13, 11, 16, 3, 3, 2, 1, 1, 0, 0),
    ("3x3s2p1-odd-c6", 3, 9, 7, 6, 3, 3, 2, 1, 1, 0, 0),
    ("3x3s1p1-odd", 2, 9, 11, 24, 3, 3, 1, 1, 1, 0, 0),
    ("3x3s1p1-odd-c3", 2, 7, 9, 3, 3, 3, 1, 1, 1, 0, 0),
    ("3x2s3-gaps", 2, 11, 10, 8, 3, 2, 3, 0, 0, 0, 0),
    ("3x2s3-gaps-pad-c5", 2, 11, 10, 5, 3, 2, 3, 1, 1, 0, 0),
    ("3x3s2-uncovered", 2, 12, 10, 8, 3, 3, 2, 0, 0, 0, 0),
    ("2x2s2-uncovered-c2", 2, 11, 13, 2, 2, 2, 2, 0, 0, 0, 0),
    ("7x7s7", 2, 15, 14, 8, 7, 7, 7, 0, 0, 0, 0),
    ("7x7s7p3-c3", 1, 14, 16, 3, 7, 7, 7, 3, 3, 0, 0),
    ("1x1s2", 2, 9, 8, 16, 1, 1, 2, 0, 0, 0, 0),
    ("1x1s2-c7", 2, 9, 8, 7, 1, 1, 2, 0, 0, 0, 0),
    ("pitched-c16", 2, 12, 12, 16, 2, 2, 2, 0, 0, 104, 9),
    ("pitched-3x3s2p1-c3", 2, 12, 10, 3, 3, 3, 2, 1, 1, 24, 8),
    ("many-ctas-128x56x56x64", 128, 56, 56, 64, 2, 2, 2, 0, 0, 0, 0),
]


def special_x(rng, shape):
    """small integers (ties) with NaN, +-Inf, +-0 and rows of -Inf (windows of all -Inf where a window is one row tall)"""
    x = rng.integers(-3, 4, shape).astype(np.float32)
    flat = x.reshape(-1)
    for v, frac in ((np.nan, 0.03), (np.inf, 0.02), (-np.inf, 0.05), (0.0, 0.05), (-0.0, 0.05)):
        flat[rng.choice(flat.size, max(1, int(frac * flat.size)), replace=False)] = v
    x[:, ::5] = -np.inf
    return x


def layout(case):
    _, N, H, W, C, R, S, st, ph, pw, pitch, rows = case
    P, Q = MR.out_size(H, W, R, S, st, ph, pw)
    return P, Q, (pitch or (Q * C + 7) // 8 * 8), (rows or P)


def run_fwd(eng, case, x_bits, with_argmax=True):
    """y in a NaN-prefilled pitched buffer [N][rows][pitch], argmax prefilled with 0xEE"""
    _, N, H, W, C, R, S, st, ph, pw, pitch, rows = case
    P, Q, pitch_u, rows_u = layout(case)
    xd = eng.to_device(x_bits)
    y = eng.to_device(np.full((N, rows_u, pitch_u), NAN_BF16, np.uint16))
    am = eng.to_device(np.full((N, P, Q, C), 0xEE, np.uint8)) if with_argmax else None
    eng.maxpool_nhwc_fwd(xd, y, am, N, H, W, C, R, S, st, (ph, pw), pitch, rows)
    eng.sync()
    return y.to_host(), (am.to_host() if with_argmax else None)


def run_bwd(eng, case, dy_img, am, pad_value=NAN_BF16):
    """dx in a NaN-prefilled dense buffer; dy written into its pitched layout with `pad_value` in the pad"""
    _, N, H, W, C, R, S, st, ph, pw, pitch, rows = case
    P, Q, pitch_u, rows_u = layout(case)
    dy = np.full((N, rows_u, pitch_u), pad_value, np.uint16)
    dy[:, :P, :Q * C] = dy_img.reshape(N, P, Q * C)
    dx = eng.to_device(np.full((N, H, W, C), NAN_BF16, np.uint16))
    eng.maxpool_nhwc_bwd(eng.to_device(dy), eng.to_device(am), dx, N, H, W, C, R, S, st, (ph, pw), pitch, rows)
    eng.sync()
    return dx.to_host()


def image(y, case):
    N, C = case[1], case[4]
    P, Q, _, _ = layout(case)
    return y[:, :P, :Q * C].reshape(N, P, Q, C)


def torch_cuda_pool(pkg, case, x_bits, dy_bits):
    """torch's CUDA max pool and its gradient on channels-last bf16 tensors holding the same bits"""
    _, N, H, W, C, R, S, st, ph, pw, _, _ = case
    xt = torch.from_numpy(x_bits.view(np.int16)).cuda().view(torch.bfloat16).permute(0, 3, 1, 2)
    y, idx = torch.nn.functional.max_pool2d(xt, (R, S), st, (ph, pw), return_indices=True)
    dyt = torch.from_numpy(dy_bits.view(np.int16)).cuda().view(torch.bfloat16).permute(0, 3, 1, 2)
    dx = torch.ops.aten.max_pool2d_with_indices_backward(dyt, xt, [R, S], [st, st], [ph, pw], [1, 1], False, idx)
    bits = lambda t: t.permute(0, 2, 3, 1).contiguous().view(torch.int16).cpu().numpy().view(np.uint16)
    return bits(y), idx.permute(0, 2, 3, 1).cpu().numpy(), bits(dx)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_pool_case(eng, pkg, case):
    _, N, H, W, C, R, S, st, ph, pw, pitch, rows = case
    P, Q, pitch_u, rows_u = layout(case)
    info = pkg.maxpool_nhwc_info(N, H, W, C, R, S, st, (ph, pw), pitch, rows)
    assert (info["P"], info["Q"], info["row_pitch"]) == (P, Q, pitch_u)
    rng = np.random.default_rng(sum(case[1:]))
    bf = pkg.f32_to_bf16_bits
    x_int = bf(rng.integers(-4, 5, (N, H, W, C)).astype(np.float32))
    for kind, x_bits in (("special", bf(special_x(rng, (N, H, W, C)))), ("integer", x_int)):
        xf = pkg.bf16_bits_to_f32(x_bits)
        a = MR.fwd_argmax(xf, R, S, st, ph, pw)
        y, am = run_fwd(eng, case, x_bits)
        # forward: argmax and y bit-identical, y = x at argmax, pad of y untouched
        assert np.array_equal(am, a), kind
        y_img = image(y, case)
        assert np.array_equal(y_img, MR.gather(x_bits, a, S, st, ph, pw)), kind
        assert np.all(y[:, :P, Q * C:] == NAN_BF16) and np.all(y[:, P:, :] == NAN_BF16)
        y0, _ = run_fwd(eng, case, x_bits, with_argmax=False)
        assert np.array_equal(y0, y)
        y1, am1 = run_fwd(eng, case, x_bits)
        assert np.array_equal(y1, y) and np.array_equal(am1, am)
        # backward: integer and random dy
        dys = {"integer": bf(rng.integers(-3, 4, (N, P, Q, C)).astype(np.float32)),
               "random": bf(rng.standard_normal((N, P, Q, C)).astype(np.float32))}
        _, cnt = MR.bwd_sum(np.ones((N, P, Q, C), np.float32), a, H, W, R, S, st, ph, pw)
        if st >= R and st >= S:
            assert cnt.max() <= 1
        for dkind, dy in dys.items():
            dx = run_bwd(eng, case, dy, am)
            want = MR.bwd_bf16(pkg, dy, a, H, W, R, S, st, ph, pw)
            assert np.array_equal(dx, want), (kind, dkind, int(np.sum(dx != want)))
            assert np.all(dx[cnt == 0] == 0)                       # +0 wherever no argmax points
            assert np.array_equal(run_bwd(eng, case, dy, am, pad_value=0), dx)    # NaN in dy's pad changes no bit
            assert np.array_equal(run_bwd(eng, case, dy, am), dx)                  # rerun
            if kind == "integer" and dkind == "integer":           # <dy, y> = <dx, x>, exact in float64
                lhs = np.sum(pkg.bf16_bits_to_f32(dy).astype(np.float64) * pkg.bf16_bits_to_f32(y_img))
                rhs = np.sum(pkg.bf16_bits_to_f32(dx).astype(np.float64) * xf)
                assert lhs == rhs
        # torch's CUDA max pool on the same channels-last bf16 tensors
        ty, tidx, tdx = torch_cuda_pool(pkg, case, x_bits, dys["random"])
        h, w = MR.winner_hw(a, S, st, ph, pw)
        ours_dx = MR.bwd_bf16(pkg, dys["random"], a, H, W, R, S, st, ph, pw)
        if kind == "integer":                                      # finite with ties: identical values and indices
            assert np.array_equal(ty, y_img) and np.array_equal(tidx, h * W + w)
            single = cnt <= 1                                      # one term or none: no order to differ in
            assert np.array_equal(tdx[single], ours_dx[single])
            n_multi, n_diff = int(np.sum(~single)), int(np.sum(tdx[~single] != ours_dx[~single]))
            print(f"{case[0]}: torch CUDA gradient differs on {n_diff} of {n_multi} elements with several terms")
            _, _, tdx_int = torch_cuda_pool(pkg, case, x_bits, dys["integer"])   # integer sums are exact in any order
            assert np.array_equal(tdx_int, MR.bwd_bf16(pkg, dys["integer"], a, H, W, R, S, st, ph, pw))
        else:                                                      # NaN, +-Inf, +-0: recorded where torch differs
            yv = pkg.bf16_bits_to_f32(y_img)
            nan_win, ninf_win = np.isnan(yv), yv == -np.inf
            val_diff = ty != y_img
            idx_diff = tidx != h * W + w
            d = idx_diff & ninf_win
            rest = ~nan_win & ~ninf_win
            print(f"{case[0]} special x vs torch CUDA: windows with NaN {int(nan_win.sum())}, value bits differ there "
                  f"{int(val_diff[nan_win].sum())}, index differs there {int(idx_diff[nan_win].sum())}; windows of all -Inf "
                  f"{int(ninf_win.sum())}, value bits differ there {int(val_diff[ninf_win].sum())}, index differs there "
                  f"{int(d.sum())} (torch {tidx[d][:4].tolist()}, first in-image element {(h * W + w)[d][:4].tolist()}); "
                  f"other windows: values differ {int(val_diff[rest].sum())}, indices {int(idx_diff[rest].sum())}")


def test_pool_refusals(eng, pkg):
    N, H, W, C, R = 2, 8, 8, 16, 2
    x = eng.array((N, H, W, C + 8), np.uint16)
    y = eng.array((N, 4, 4 * C + 8), np.uint16)
    am = eng.array((N, 4, 4, C + 8), np.uint8)
    dx = eng.array((N, H, W, C + 8), np.uint16)
    fwd = lambda *a, **k: eng.maxpool_nhwc_fwd(*a, **k)
    bwd = lambda *a, **k: eng.maxpool_nhwc_bwd(*a, **k)
    shape = (N, H, W, C, R, R, R)
    cases = [
        (lambda: fwd(x, y, am, N, H, W, C, 8, 2, 2), "pcnn_maxpool_nhwc_bf16_fwd: 8x2 window: 1 <= R, S <= 7"),
        (lambda: fwd(x, y, am, 0, H, W, C, 2, 2, 2), "each must be >= 1"),
        (lambda: fwd(x, y, am, N, H, W, C, 2, 2, 8), "1 <= stride <= 7"),
        (lambda: fwd(x, y, am, N, H, W, C, 3, 3, 2, (2, 0)), "pad_h <= R/2"),
        (lambda: fwd(x, y, am, N, 1, W, C, 5, 2, 2, (2, 0)), None),
        (lambda: fwd(x, y, am, N, 1, W, C, 7, 2, 2, (2, 0)), "H \\+ 2 pad_h >= R"),
        (lambda: fwd(x, y, am, *shape, row_pitch=60), "row_pitch 60"),
        (lambda: fwd(x, y, am, *shape, image_rows=3), "image_rows 3"),
        (lambda: bwd(y, am, dx, N, H, W, C, 2, 2, 2, (0, 2)), "pcnn_maxpool_nhwc_bf16_bwd: padding \\(0, 2\\)"),
        (lambda: bwd(y, am, dx, *shape, row_pitch=68), "multiple of 8"),
        (lambda: fwd(None, y, am, *shape), "NULL context, x or y"),
        (lambda: fwd(x, None, am, *shape), "NULL context, x or y"),
        (lambda: bwd(None, am, dx, *shape), "NULL context, dy, argmax or dx"),
        (lambda: bwd(y, None, dx, *shape), "NULL context, dy, argmax or dx"),
        (lambda: bwd(y, am, None, *shape), "NULL context, dy, argmax or dx"),
        (lambda: fwd(x.ptr + 2, y, am, *shape), "16-byte aligned"),
        (lambda: fwd(x, y.ptr + 8, am, *shape), "16-byte aligned"),
        (lambda: fwd(x, y, am.ptr + 8, *shape), "16-byte aligned"),
        (lambda: bwd(y.ptr + 4, am, dx, *shape), "16-byte aligned"),
        (lambda: bwd(y, am.ptr + 1, dx, *shape), "16-byte aligned"),
        (lambda: bwd(y, am, dx.ptr + 2, *shape), "16-byte aligned"),
        (lambda: fwd(x, x.ptr + 64, am, *shape), "overlapping buffers"),
        (lambda: fwd(x, y, x.ptr + 1024, *shape), "overlapping buffers"),
        (lambda: fwd(x, y, y.ptr + 16, *shape), "overlapping buffers"),
        (lambda: bwd(y, am, y, *shape), "overlapping buffers"),
        (lambda: bwd(y, dx.ptr + 256, dx, *shape), "overlapping buffers"),
    ]
    for fn, msg in cases:
        if msg is None:
            fn()
            continue
        with pytest.raises(pkg.PcnnError, match=msg):
            fn()
    fwd(x, y, None, *shape)                                        # argmax NULL is inference
    eng.sync()


def test_stack_conv_pool_conv_pool(eng, pkg, golden):
    """ConvLayer 28x28x1 -> 8@5x5 sigmoid + bias (row-Toeplitz), MaxPoolLayer 2x2 into the next layer's pitched x, ConvLayer
    12x12x8 -> 16@3x3 padding 1 + bias (wide), MaxPoolLayer 2x2, loss 1/2 |y - t|^2, on 64 MNIST digits.  In each of the first 5
    steps both pools are bit-identical to the numpy reference on the device's own tensors, and dw, db of both layers are within
    the bounds of test_conv_train_gpu.py::test_layer_step_sigmoid_random against float64 on the device's intermediates (fp32
    accumulation within 2 n 2^-24 sum |terms|, n = output pixels).  The loss falls over 20 SGD steps."""
    B = 64
    rng = np.random.default_rng(77)
    f1, b1 = rng.uniform(-0.2, 0.2, (8, 5, 5, 1)).astype(np.float32), rng.uniform(-0.2, 0.2, 8).astype(np.float32)
    f2, b2 = rng.uniform(-0.1, 0.1, (16, 3, 3, 8)).astype(np.float32), rng.uniform(-0.1, 0.1, 16).astype(np.float32)
    l1 = pkg.ConvLayer(eng, B, 28, 28, 1, 8, 5, 5, f1, b1, act=1)
    l2 = pkg.ConvLayer(eng, B, 12, 12, 8, 16, 3, 3, f2, b2, act=0, padding=(1, 1), row_pitch=104)
    p1 = pkg.MaxPoolLayer(eng, B, 24, 24, 8, 2, row_pitch=l2.row_pitch, image_rows=l2.image_rows)
    p2 = pkg.MaxPoolLayer(eng, B, 12, 12, 16, 2)
    assert (l1.family, l2.family) == ("narrow", "wide")
    assert p1.out_shape == (B, 12, 12, 8) and p1.row_pitch == 104 and p2.out_shape == (B, 6, 6, 16) and p2.row_pitch == 96
    imgs = golden["train_u8"][:B].reshape(B, 28, 28).astype(np.float32) / 255.0
    xl = np.zeros((B * 28, 32), np.uint16)
    xl[:, :28] = pkg.f32_to_bf16_bits(imgs).reshape(B * 28, 28)
    xd = eng.to_device(xl)
    x1 = pkg.bf16_bits_to_f32(xl[:, :28]).reshape(B, 28, 28, 1).astype(np.float64)
    dev = torch.device("cuda", 0)
    y1, dy1 = (torch.full((B, 24, 24, 8), NAN_BF16, dtype=torch.int16, device=dev) for _ in range(2))
    x2, dx2 = (torch.full((B, 12, 104), NAN_BF16, dtype=torch.int16, device=dev) for _ in range(2))
    y2, dy2 = (torch.full((B, 12, 12, 16), NAN_BF16, dtype=torch.int16, device=dev) for _ in range(2))
    y3, dy3 = (torch.full((B, 6, 96), NAN_BF16, dtype=torch.int16, device=dev) for _ in range(2))
    t = torch.from_numpy(rng.uniform(0, 1, (B, 6, 6, 16)).astype(np.float32)).to(dev)
    host = lambda a: a.cpu().numpy().view(np.uint16) if isinstance(a, torch.Tensor) else a.to_host()
    f32 = pkg.bf16_bits_to_f32
    losses = []
    for it in range(20):
        check = it < 5
        l1.forward(xd, y1)
        p1.forward(y1, x2)
        l2.forward(x2, y2)
        p2.forward(y2, y3)
        eng.sync()
        e = y3.view(torch.bfloat16).float().reshape(B, 6, 6, 16) - t
        dy3.view(torch.bfloat16).copy_(e.reshape(B, 6, 96).to(torch.bfloat16))
        losses.append(0.5 * float((e.double() ** 2).sum()))
        torch.cuda.synchronize()
        if check:
            h = {k: host(v) for k, v in dict(y1=y1, x2=x2, y2=y2, y3=y3, dy3=dy3, am1=p1.argmax, am2=p2.argmax).items()}
        p2.backward(dy3, dy2)
        if check:
            eng.sync()
            h["dy2"] = host(dy2)                                   # before l2.backward turns it into dpre in place
        l2.backward(y2, dy2, dx2)
        if check:
            eng.sync()
            h["dpre2"], h["dx2"] = host(dy2), host(dx2)
        p1.backward(dx2, dy1)
        if check:
            eng.sync()
            h["dy1"] = host(dy1)
        l1.backward(y1, dy1, None)
        if check:
            eng.sync()
            h["dpre1"] = host(dy1)
            dw1, db1, dw2, db2 = (a.to_host() for a in (l1.dw, l1.db, l2.dw, l2.db))
            # pool 1: y1 -> x2 (pitched), dx2 (pitched, its pad columns never written: NaN) -> dy1
            a1 = MR.fwd_argmax(f32(h["y1"]), 2, 2, 2, 0, 0)
            assert np.array_equal(h["am1"], a1), it
            assert np.array_equal(h["x2"][:, :, :96].reshape(B, 12, 12, 8), MR.gather(h["y1"], a1, 2, 2, 0, 0)), it
            assert np.array_equal(h["dy1"], MR.bwd_bf16(pkg, h["dx2"][:, :, :96].reshape(B, 12, 12, 8), a1, 24, 24, 2, 2, 2, 0, 0)), it
            # pool 2: y2 -> y3, dy3 -> dy2
            a2 = MR.fwd_argmax(f32(h["y2"]), 2, 2, 2, 0, 0)
            assert np.array_equal(h["am2"], a2), it
            assert np.array_equal(h["y3"].reshape(B, 6, 6, 16), MR.gather(h["y2"], a2, 2, 2, 0, 0)), it
            assert np.array_equal(h["dy2"], MR.bwd_bf16(pkg, h["dy3"].reshape(B, 6, 6, 16), a2, 12, 12, 2, 2, 2, 0, 0)), it
            # dw, db of both layers against float64 on the device's intermediates
            x2f = np.pad(f32(h["x2"][:, :, :96]).reshape(B, 12, 12, 8).astype(np.float64), ((0, 0), (1, 1), (1, 1), (0, 0)))
            for dw, db, xin, dpre, R in ((dw1, db1, x1, h["dpre1"], 5), (dw2, db2, x2f, h["dpre2"], 3)):
                d = f32(dpre).astype(np.float64)
                npix = d.shape[0] * d.shape[1] * d.shape[2]
                ref, ref_abs = CS.conv_wgrad_f64(xin, d, R, R, 1), CS.conv_wgrad_f64(np.abs(xin), np.abs(d), R, R, 1)
                assert np.all(np.abs(dw - ref) <= 2 * npix * 2.0 ** -24 * ref_abs + 1e-30), it
                assert np.all(np.abs(db - d.sum(axis=(0, 1, 2))) <= 2 * npix * 2.0 ** -24 * np.abs(d).sum(axis=(0, 1, 2))), it
        l1.sgd(LR)
        l2.sgd(LR)
        eng.sync()
    for layer in (l1, l2, p1, p2):
        layer.close()
    print("loss over 20 steps:", " ".join(f"{v:.4g}" for v in losses))
    assert losses[-1] < losses[0]
