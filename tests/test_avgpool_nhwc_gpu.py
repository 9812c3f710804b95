"""The NHWC average pools on the device (pcnn_avgpool_nhwc_bf16_fwd / _bwd, pcnn_global_avgpool_nhwc_bf16_fwd / _bwd, AvgPoolLayer,
GlobalAvgPoolLayer): windowed y and dx and global dx bit-identical to the float32 replays of tests/avgpool_ref.py (pinned to
torch's CPU float64 pools by test_avgpool_nhwc_cpu.py), global y exact on integer operands and within an error model on random
ones, torch's CUDA pools on the same channels-last bf16 tensors recorded, every refusal, and a ResNet with a projection block and a
global-average-pool head trained on MNIST digits.

Error model of the global forward (random operands).  With n_acc = (pixels per lane - 1) + (lanes - 1) + (ranges - 1) additions on
the longest path of the partition global_avgpool_nhwc_info reports, u = 2^-24, gamma = n_acc u / (1 - n_acc u), S the exact sum of
an image's channel and A the sum of its absolute values: |s - S| <= gamma A, and the quotient q = fl(s / HW) satisfies
|q - S / HW| <= E = (gamma A + u (|S| + gamma A)) / HW.  bf16 rounding is monotonic, so y lies between bf16_rn(S/HW - E) and
bf16_rn(S/HW + E)."""
import numpy as np
import pytest
import torch

import avgpool_ref as AR
import maxpool_ref as MR
from avgpool_ref import gap_bound
from example_nets import DEV, NAN_BF16, ResNetGAP, host, train

pytestmark = pytest.mark.gpu

U = 2.0 ** -24

CASES = [  # id, N, H, W, C, R, S, stride, pad_h, pad_w, row_pitch (0 = Q*C rounded up to 8), image_rows (0 = P)
    ("c1-2x2s2", 2, 10, 9, 1, 2, 2, 2, 0, 0, 0, 0),
    ("c3-2x2s2", 2, 10, 9, 3, 2, 2, 2, 0, 0, 0, 0),
    ("c6-2x2s2-pitched", 3, 24, 24, 6, 2, 2, 2, 0, 0, 80, 14),
    ("c16-2x2s2", 2, 10, 9, 16, 2, 2, 2, 0, 0, 0, 0),
    ("c64-3x3s1p1", 2, 9, 11, 64, 3, 3, 1, 1, 1, 0, 0),
    ("c256-2x2s2", 2, 10, 9, 256, 2, 2, 2, 0, 0, 0, 0),
    ("c320-3x3s2p1-odd", 2, 9, 7, 320, 3, 3, 2, 1, 1, 0, 0),
    ("c16-3x3s2p1-odd", 2, 13, 11, 16, 3, 3, 2, 1, 1, 0, 0),
    ("c6-3x3s2p1-odd", 3, 9, 7, 6, 3, 3, 2, 1, 1, 0, 0),
    ("c3-3x3s1p1-odd", 2, 7, 9, 3, 3, 3, 1, 1, 1, 0, 0),
    ("c8-3x2s3-gaps", 2, 11, 10, 8, 3, 2, 3, 0, 0, 0, 0),
    ("c6-3x2s3-gaps-pad", 2, 11, 10, 6, 3, 2, 3, 1, 1, 0, 0),
    ("c16-7x7s7", 2, 15, 14, 16, 7, 7, 7, 0, 0, 0, 0),
    ("c3-7x7s7p3", 1, 14, 16, 3, 7, 7, 7, 3, 3, 0, 0),
    ("c1-1row-1x3s1p1", 3, 1, 9, 1, 1, 3, 1, 0, 1, 0, 0),
    ("c16-pitched-3x3s2p1", 2, 12, 12, 16, 3, 3, 2, 1, 1, 104, 9),
    ("many-ctas-128x56x56x64", 128, 56, 56, 64, 2, 2, 2, 0, 0, 0, 0),
]


def same_or_nan(got, want):
    """bf16 bits: identical where want is a number; NaN (any payload) where want is NaN"""
    nan, gnan = (want & 0x7FFF) > 0x7F80, (got & 0x7FFF) > 0x7F80
    return np.array_equal(gnan, nan) and np.array_equal(got[~nan], want[~nan])


def special_x(rng, shape):
    """normal values with NaN, +-Inf and +-0 sprinkled in, and rows of -0"""
    x = rng.standard_normal(shape).astype(np.float32)
    flat = x.reshape(-1)
    for v, frac in ((np.nan, 0.01), (np.inf, 0.01), (-np.inf, 0.01), (0.0, 0.05), (-0.0, 0.05)):
        flat[rng.choice(flat.size, max(1, int(frac * flat.size)), replace=False)] = v
    x[:, ::4] = -0.0
    return x


def layout(case):
    _, N, H, W, C, R, S, st, ph, pw, pitch, rows = case
    P, Q = MR.out_size(H, W, R, S, st, ph, pw)
    return P, Q, (pitch or (Q * C + 7) // 8 * 8), (rows or P)


def run_fwd(eng, case, cip, x_bits):
    _, N, H, W, C, R, S, st, ph, pw, pitch, rows = case
    P, Q, pitch_u, rows_u = layout(case)
    y = eng.to_device(np.full((N, rows_u, pitch_u), NAN_BF16, np.uint16))
    eng.avgpool_nhwc_fwd(eng.to_device(x_bits), y, N, H, W, C, R, S, st, (ph, pw), cip, pitch, rows)
    eng.sync()
    return y.to_host()


def run_bwd(eng, case, cip, dy_img, pad_value=NAN_BF16):
    _, N, H, W, C, R, S, st, ph, pw, pitch, rows = case
    P, Q, pitch_u, rows_u = layout(case)
    dy = np.full((N, rows_u, pitch_u), pad_value, np.uint16)
    dy[:, :P, :Q * C] = dy_img.reshape(N, P, Q * C)
    dx = eng.to_device(np.full((N, H, W, C), NAN_BF16, np.uint16))
    eng.avgpool_nhwc_bwd(eng.to_device(dy), dx, N, H, W, C, R, S, st, (ph, pw), cip, pitch, rows)
    eng.sync()
    return dx.to_host()


def cuda_bf16(bits):
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).to(DEV).view(torch.bfloat16).permute(0, 3, 1, 2)


def host_bits(t):
    return t.permute(0, 2, 3, 1).contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


@pytest.mark.parametrize("cip", [0, 1])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_windowed(eng, pkg, case, cip):
    _, N, H, W, C, R, S, st, ph, pw, pitch, rows = case
    P, Q, pitch_u, rows_u = layout(case)
    assert pkg.avgpool_nhwc_info(N, H, W, C, R, S, st, (ph, pw), pitch, rows)["row_pitch"] == pitch_u
    rng = np.random.default_rng(sum(case[1:]) + cip)
    bf, f32 = pkg.f32_to_bf16_bits, pkg.bf16_bits_to_f32
    img = lambda y: y[:, :P, :Q * C].reshape(N, P, Q, C)
    cnt = AR.counts(H, W, R, S, st, ph, pw, cip)
    pow2 = bool(np.all((cnt & (cnt - 1)) == 0))
    for kind, x_bits in (("random", bf(rng.standard_normal((N, H, W, C)).astype(np.float32))), ("special", bf(special_x(rng, (N, H, W, C)))),
                         ("integer", bf(rng.integers(-4, 5, (N, H, W, C)).astype(np.float32)))):
        y = run_fwd(eng, case, cip, x_bits)
        want = bf(AR.fwd(f32(x_bits), R, S, st, ph, pw, cip))
        assert same_or_nan(img(y), want), (kind, int(np.sum(img(y) != want)))
        assert np.all(y[:, :P, Q * C:] == NAN_BF16) and np.all(y[:, P:, :] == NAN_BF16)          # pad untouched
        assert np.array_equal(run_fwd(eng, case, cip, x_bits), y)                               # rerun
        if kind == "special":
            continue
        dy = bf(rng.integers(-3, 4, (N, P, Q, C)).astype(np.float32) if kind == "integer" else rng.standard_normal((N, P, Q, C)).astype(np.float32))
        dx = run_bwd(eng, case, cip, dy)
        want_dx, terms = AR.bwd(f32(dy), H, W, R, S, st, ph, pw, cip)
        assert np.array_equal(dx, bf(want_dx)), (kind, int(np.sum(dx != bf(want_dx))))
        assert np.all(dx[:, terms == 0] == 0)                                                   # +0 with no term
        assert np.array_equal(run_bwd(eng, case, cip, dy, pad_value=0), dx)                     # NaN in dy's pad changes no bit
        assert np.array_equal(run_bwd(eng, case, cip, dy), dx)                                  # rerun
        if kind == "integer" and pow2:                                                          # exact adjoint: <y, dy> = <x, dx>
            lhs = np.sum(f32(dy).astype(np.float64) * f32(img(y)))
            rhs = np.sum(f32(dx).astype(np.float64) * f32(x_bits))
            assert lhs == rhs
        if kind == "random":                                                                    # torch CUDA, recorded
            xt = cuda_bf16(x_bits).requires_grad_(True)
            ty = torch.nn.functional.avg_pool2d(xt, (R, S), st, (ph, pw), count_include_pad=bool(cip))
            ty.backward(cuda_bf16(dy))
            print(f"{case[0]} cip={cip} vs torch CUDA: y bits differ on {int(np.sum(host_bits(ty.detach()) != img(y)))} of {img(y).size}, "
                  f"dx on {int(np.sum(host_bits(xt.grad) != dx))} of {dx.size}")
    # the layer drives the same calls
    layer = pkg.AvgPoolLayer(eng, N, H, W, C, R, S, st, (ph, pw), bool(cip), pitch or None, rows)
    assert layer.out_shape == (N, P, Q, C) and layer.row_pitch == pitch_u


GSHAPES = [(3, H, W, C) for C in (1, 6, 8, 300, 2048) for H, W in ((1, 1), (7, 7), (56, 56))] + [(8, 56, 56, 256)]


@pytest.mark.parametrize("shape", GSHAPES, ids=["x".join(map(str, s)) for s in GSHAPES])
def test_global(eng, pkg, shape):
    N, H, W, C = shape
    rng = np.random.default_rng(sum(shape))
    bf, f32 = pkg.f32_to_bf16_bits, pkg.bf16_bits_to_f32
    for pitch in (0, (C + 7) // 8 * 8 + 8):
        info = pkg.global_avgpool_nhwc_info(N, H, W, C, pitch)
        pu = info["row_pitch"]
        layer = pkg.GlobalAvgPoolLayer(eng, N, H, W, C, pitch or None)
        assert layer.info == info

        def fwd(x_bits):
            y = eng.to_device(np.full((N, pu), NAN_BF16, np.uint16))
            layer.forward(eng.to_device(x_bits), y)
            eng.sync()
            return y.to_host()

        x_int = bf(rng.integers(-8, 9, shape).astype(np.float32))
        y = fwd(x_int)
        assert np.array_equal(y[:, :C], bf(AR.global_fwd(f32(x_int), info)))                   # exact sums
        assert np.all(y[:, C:] == NAN_BF16)
        x_rnd = bf((rng.standard_normal(shape) + 0.5).astype(np.float32))
        y = fwd(x_rnd)
        m, E, lo, hi = gap_bound(pkg, f32(x_rnd), info)
        yf = f32(y[:, :C])
        assert np.all((yf >= lo) & (yf <= hi))
        ulp = np.maximum(np.abs(m), 2.0 ** -126) * 2.0 ** -8
        ratio = float(np.max(np.abs(yf - m) / (E + ulp / 2)))
        diff = int(np.sum(y[:, :C] != bf(AR.global_fwd(f32(x_rnd), info))))
        print(f"GAP {shape} pitch {pu}: {info['ranges']} ranges, {info['ctas']} CTAs; worst |y - mean| / (E + half bf16 ulp) {ratio:.3f}; "
              f"bits differing from the ordered float32 replay {diff}")
        assert np.array_equal(fwd(x_rnd), y)                                                    # rerun
        dy_img = bf(rng.standard_normal((N, C)).astype(np.float32))
        dy = np.full((N, pu), NAN_BF16, np.uint16)
        dy[:, :C] = dy_img
        dx = eng.to_device(np.full((N, H, W, C), NAN_BF16, np.uint16))
        layer.backward(eng.to_device(dy), dx)
        eng.sync()
        assert np.array_equal(dx.to_host(), bf(AR.global_bwd(f32(dy_img), H, W)))             # every pixel written, pad never read
        if pitch == 0 and N * H * W * C < 1 << 24:                                              # torch CUDA, recorded
            xt = cuda_bf16(x_rnd.reshape(shape))
            ty = xt.mean((2, 3)).contiguous().view(torch.int16).cpu().numpy().view(np.uint16)
            ta = torch.nn.functional.adaptive_avg_pool2d(xt, 1)[:, :, 0, 0].contiguous().view(torch.int16).cpu().numpy().view(np.uint16)
            print(f"GAP {shape} vs torch CUDA: mean differs on {int(np.sum(ty != y[:, :C]))}, adaptive_avg_pool2d on "
                  f"{int(np.sum(ta != y[:, :C]))} of {N * C}")


def test_refusals(eng, pkg):
    N, H, W, C = 2, 8, 8, 16
    x = eng.array((N, H, W, C + 8), np.uint16)
    y = eng.array((N, 4, 4 * C + 8), np.uint16)
    dx = eng.array((N, H, W, C + 8), np.uint16)
    fwd, bwd = eng.avgpool_nhwc_fwd, eng.avgpool_nhwc_bwd
    gf, gb = eng.global_avgpool_nhwc_fwd, eng.global_avgpool_nhwc_bwd
    shape = (N, H, W, C, 2, 2, 2)
    cases = [
        (lambda: fwd(x, y, N, H, W, C, 8, 2, 2), "pcnn_avgpool_nhwc_bf16_fwd: 8x2 window: 1 <= R, S <= 7"),
        (lambda: fwd(x, y, 0, H, W, C, 2, 2, 2), "each must be >= 1"),
        (lambda: fwd(x, y, N, H, W, C, 2, 2, 8), "1 <= stride <= 7"),
        (lambda: fwd(x, y, N, H, W, C, 3, 3, 2, (2, 0)), "pad_h <= R/2"),
        (lambda: fwd(x, y, N, 1, W, C, 7, 2, 2, (2, 0)), "H \\+ 2 pad_h >= R"),
        (lambda: fwd(x, y, *shape, row_pitch=60), "row_pitch 60"),
        (lambda: fwd(x, y, *shape, image_rows=3), "image_rows 3"),
        (lambda: fwd(x, y, *shape, count_include_pad=2), "pcnn_avgpool_nhwc_bf16_fwd: count_include_pad = 2: 0 or 1"),
        (lambda: bwd(y, dx, *shape, count_include_pad=-1), "pcnn_avgpool_nhwc_bf16_bwd: count_include_pad = -1: 0 or 1"),
        (lambda: bwd(y, dx, N, H, W, C, 2, 2, 2, (0, 2)), "pcnn_avgpool_nhwc_bf16_bwd: padding \\(0, 2\\)"),
        (lambda: bwd(y, dx, *shape, row_pitch=68), "multiple of 8"),
        (lambda: fwd(None, y, *shape), "NULL context, x or y"),
        (lambda: fwd(x, None, *shape), "NULL context, x or y"),
        (lambda: bwd(None, dx, *shape), "NULL context, dy or dx"),
        (lambda: bwd(y, None, *shape), "NULL context, dy or dx"),
        (lambda: fwd(x.ptr + 2, y, *shape), "16-byte aligned"),
        (lambda: fwd(x, y.ptr + 8, *shape), "16-byte aligned"),
        (lambda: bwd(y.ptr + 4, dx, *shape), "16-byte aligned"),
        (lambda: bwd(y, dx.ptr + 2, *shape), "16-byte aligned"),
        (lambda: fwd(x, x.ptr + 64, *shape), "overlapping buffers"),
        (lambda: bwd(y, y, *shape), "overlapping buffers"),
        (lambda: gf(x, y, 0, H, W, C), "pcnn_global_avgpool_nhwc_bf16_fwd: N = 0, H = 8, W = 8, C = 16: each must be >= 1"),
        (lambda: gb(y, dx, N, H, 0, C), "pcnn_global_avgpool_nhwc_bf16_bwd: .* each must be >= 1"),
        (lambda: gf(x, y, N, 46341, 46341, 1), "32-bit index range"),
        (lambda: gf(x, y, N, H, W, C, row_pitch=12), "row_pitch 12: 0 \\(C rounded up to 8\\) or a multiple of 8"),
        (lambda: gb(y, dx, N, H, W, C, row_pitch=8), "row_pitch 8"),
        (lambda: gf(None, y, N, H, W, C), "NULL context, x or y"),
        (lambda: gb(y, None, N, H, W, C), "NULL context, dy or dx"),
        (lambda: gf(x.ptr + 2, y, N, H, W, C), "16-byte aligned"),
        (lambda: gb(y, dx.ptr + 8, N, H, W, C), "16-byte aligned"),
        (lambda: gf(x, x.ptr + 32, N, H, W, C), "overlapping buffers"),
        (lambda: gb(dx.ptr + 64, dx, N, H, W, C), "overlapping buffers"),
    ]
    for fn, msg in cases:
        with pytest.raises(pkg.PcnnError, match=msg):
            fn()
    fwd(x, y, *shape)
    gf(x, y, N, H, W, C)
    eng.sync()


# ------------------------------------------------------------------------------------------------ end to end
ACC_MIN = 0.88          # a float32 torch CPU replica of this network, initialisation and step reaches 0.949 (DESIGN 3.16)


def test_resnet_gap_mnist(eng, pkg, golden):
    """In each of the first 5 steps the avg pool's y and dx and GAP's dx are bit-exact against the replays on the device's own
    tensors, and GAP's y lies within its error model.  A fresh run reproduces the parameters after 5 steps bit for bit.  After
    EPOCHS epochs over the 1024 training digits the mean loss has fallen, and test accuracy on the 256 test digits, evaluated with
    the running statistics, exceeds ACC_MIN."""
    bf, f32 = pkg.f32_to_bf16_bits, pkg.bf16_bits_to_f32
    NB = ResNetGAP.NB

    def check_step(net, it, x, labels):
        net.forward(x, labels)
        eng.sync()
        z1, x2, out, h = host(net.z1), host(net.x2), host(net.out), host(net.h)
        net.backward()
        eng.sync()
        assert np.array_equal(x2[:, :, :96].reshape(NB, 12, 12, 8), bf(AR.fwd(f32(z1), 2, 2, 2, 0, 0, 1))), it
        dx2 = host(net.dx2)[:, :, :96].reshape(NB, 12, 12, 8)
        assert np.array_equal(host(net.dz1), bf(AR.bwd(f32(dx2), 24, 24, 2, 2, 2, 0, 0, 1)[0])), it
        assert np.array_equal(host(net.dout), bf(AR.global_bwd(f32(host(net.dh)[:, :32]), 6, 6))), it
        _, _, lo, hi = gap_bound(pkg, f32(out).reshape(NB, 6, 6, 32), net.gap.info)
        yf = f32(h[:, :32])
        assert np.all((yf >= lo) & (yf <= hi)), it

    ep_loss, acc, _ = train(eng, pkg, golden, lambda: ResNetGAP(eng, pkg, ResNetGAP.init_params()), ResNetGAP.EPOCHS, check_step=check_step)
    print(f"GAP ResNet: mean loss by epoch {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}; test accuracy {acc:.4f} (threshold {ACC_MIN})")
    assert np.isfinite(ep_loss).all() and ep_loss[-1] < ep_loss[0]
    assert acc > ACC_MIN
