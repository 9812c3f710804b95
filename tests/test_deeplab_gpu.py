"""DeepLabLite (tests/deeplab_nets.py) trained on the device with segment_nets' harness: in each of the first five steps every
dilated layer is checked on its own operands against dilated_ref's float64 passes; a fresh run reproduces the parameters after five
steps bit for bit; and the test mIoU after training is within 0.05 of the float32 replica's (scripts/deeplab_replica.py)."""
import numpy as np
import pytest

import deeplab_nets
import dilated_ref as D
from example_nets import host
import segment_nets

pytestmark = pytest.mark.gpu

REPLICA_MIOU = 0.7549   # scripts/deeplab_replica.py


def _f64(pkg, buf, shape):
    return pkg.bf16_bits_to_f32(host(buf)).reshape(shape).astype(np.float64)


def check_dilated(pkg, layer, x, y, dy, dx):
    """a dilated ConvLayer or DepthwiseConvLayer (no bias, no activation) on its own bf16 operands and master: y and dx within bf16
    rounding plus an fp32 accumulation bound of the sum of |terms|, dw within the fp32 bound of its sum over N P Q pixels"""
    depthwise = isinstance(layer, pkg.DepthwiseConvLayer)
    if depthwise:
        N, H, W, C, R, S = layer.shape
        K = C
    else:
        N, H, W, C, K, R, S = layer.shape
    st, pad, dil = layer.stride, layer.padding, layer.dilation
    P, Q = D.out_size(H, W, R, S, st, pad, dil)
    xq, dyq = _f64(pkg, x, (N, H, W, C)), _f64(pkg, dy, (N, P, Q, K))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(layer.filt.to_host())).astype(np.float64)
    if depthwise:
        f = f.reshape(C, R, S)
        fwd = lambda a, b: D.dw_fwd(a, b, None, st, pad, dil)
        wgrad = lambda a, b: D.dw_wgrad_f64(a, b, R, S, st, pad, dil)
        dgrad = lambda a, b: D.dw_dgrad(a, b, H, W, st, pad, dil)
    else:
        f = f.reshape(K, R, S, C)
        fwd = lambda a, b: D.fwd_f64(a, b, None, st, pad, dil)
        wgrad = lambda a, b: D.wgrad_f64(a, b, R, S, st, pad, dil)
        dgrad = lambda a, b: D.dgrad_f64(a, b, H, W, st, pad, dil)
    ref, mag = fwd(xq, f), fwd(np.abs(xq), np.abs(f))
    assert np.all(np.abs(_f64(pkg, y, ref.shape) - ref) <= 2 ** -8 * np.abs(ref) + 2 ** -18 * mag + 1e-30), "y"
    ref, mag = dgrad(dyq, f), dgrad(np.abs(dyq), np.abs(f))
    assert np.all(np.abs(_f64(pkg, dx, ref.shape) - ref) <= 2 ** -8 * np.abs(ref) + 2 ** -18 * mag + 1e-30), "dx"
    ref, mag = wgrad(xq, dyq), wgrad(np.abs(xq), np.abs(dyq))
    got = layer.dw.to_host().reshape(ref.shape).astype(np.float64)
    assert np.all(np.abs(got - ref) <= (N * P * Q * 2.0 ** -24 + 2.0 ** -20) * mag + 1e-30), "dw"


def test_deeplab_trains(eng, pkg, golden):
    """five checked steps, a bit-identical fresh run, and the trained test mIoU near the float32 replica's (and above twice the
    all-background score)"""
    checked = []

    def check_step(net, it, x, labels, masks):
        net.forward(x, labels, masks)
        net.backward()
        eng.sync()
        for layer, xin, y, dy, dx in net.dilated():
            check_dilated(pkg, layer, xin, y, dy, dx)
        checked.append(it)

    losses, miou, bg, _ = segment_nets.train_segmenter(eng, pkg, golden, deeplab_nets.DeepLabLite, check_step)
    print(f"DeepLabLite: epoch losses {losses}, test mIoU {miou:.4f} (replica {REPLICA_MIOU:.4f}), all-background mIoU {bg:.4f}")
    assert checked == [0, 1, 2, 3, 4]
    assert losses[-1] < losses[0]
    assert abs(miou - REPLICA_MIOU) <= 0.05 and miou > 2 * bg
    _, again, _, _ = segment_nets.train_segmenter(eng, pkg, golden, deeplab_nets.DeepLabLite)
    assert again == miou
