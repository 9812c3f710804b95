"""numpy reference of the ReLU activation (PCNN_ACT_RELU) of the forward epilogues and of pcnn_conv_bias_act_bwd at act 3.
test_relu_cpu.py pins it to torch.relu and torch's threshold_backward.

Forward: y = bf16_rn(v < 0 ? +0 : v) for the fp32 pre-activation v (NaN and -0 unchanged, one rounding after the ReLU).
Backward: dpre = float(y) <= 0 ? +0 : dy, dy's bits passed through (a NaN y passes dy)."""
import numpy as np


def relu(v):
    """v < 0 ? +0 : v in v's dtype: NaN and -0 pass unchanged (torch.relu, clamp_min(0)), unlike np.maximum(v, 0)"""
    v = np.asarray(v)
    return np.where(v < 0, np.zeros((), v.dtype), v)


def fwd_bits(pkg, v):
    """bf16 bits of the epilogue's y for the fp32 pre-activation v (float32, or float64 that is exact in float32)"""
    return pkg.f32_to_bf16_bits(relu(np.asarray(v, np.float32)))


def bwd_bits(pkg, y_bits, dy_bits):
    """dpre bits of pcnn_conv_bias_act_bwd at act 3 from the bf16 bits of y and dy"""
    y = pkg.bf16_bits_to_f32(y_bits)
    with np.errstate(invalid="ignore"):
        return np.where(y <= 0, np.uint16(0), np.asarray(dy_bits, np.uint16)).astype(np.uint16)
