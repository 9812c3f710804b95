"""Replays of the optimizer rules of include/pcnn.h (pcnn_optim_*): sgd32 / adamw32 in numpy float32, one rounding per operation in
exactly the order of the header (the device must match them bit for bit), and sgd64 / adamw64, the same formulas in float64 with the
hyperparameters as Python floats (what torch.optim computes in float64).  Each takes and returns host arrays and leaves its inputs
alone; t is the step number, 1 on the first call."""
import math

import numpy as np

f32 = np.float32


def sgd32(p, g, b, lr, t, momentum=0.0, dampening=0.0, nesterov=False, wd=0.0):
    """one SGD step in float32: returns (p, b); b is None when momentum == 0"""
    lr, mu, wd = f32(lr), f32(momentum), f32(wd)
    with np.errstate(all="ignore"):
        gp = g + wd * p if wd != 0 else g.copy()
        if mu != 0:
            b = gp.copy() if t == 1 else mu * b + f32(1.0 - float(f32(dampening))) * gp
            d = gp + mu * b if nesterov else b
        else:
            b, d = None, gp
        return p + (-lr) * d, b


def adamw32(p, g, m, v, lr, t, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.0):
    """one AdamW step in float32: returns (p, m, v).  c2, s and lambda formed in double, as the host does"""
    lr, b1, b2, eps, wd = f32(lr), f32(beta1), f32(beta2), f32(eps), f32(wd)
    c2 = f32(math.sqrt(1.0 - float(b2) ** t))
    s = f32(float(lr) / (1.0 - float(b1) ** t))
    with np.errstate(all="ignore"):
        if wd != 0:
            p = p * f32(1.0 - float(lr) * float(wd))
        m = m + f32(1.0 - float(b1)) * (g - m)
        v = b2 * v + (f32(1.0 - float(b2)) * g) * g
        den = np.sqrt(v) / c2 + eps
        return p + (-s) * (m / den), m, v


def sgd64(p, g, b, lr, t, momentum=0.0, dampening=0.0, nesterov=False, wd=0.0):
    """sgd32's formulas in float64"""
    gp = g + wd * p if wd != 0 else g.copy()
    if momentum != 0:
        b = gp.copy() if t == 1 else momentum * b + (1.0 - dampening) * gp
        d = gp + momentum * b if nesterov else b
    else:
        b, d = None, gp
    return p - lr * d, b


def adamw64(p, g, m, v, lr, t, beta1=0.9, beta2=0.999, eps=1e-8, wd=0.0):
    """adamw32's formulas in float64"""
    if wd != 0:
        p = p * (1.0 - lr * wd)
    m = m + (1.0 - beta1) * (g - m)
    v = beta2 * v + ((1.0 - beta2) * g) * g
    den = np.sqrt(v) / math.sqrt(1.0 - beta2 ** t) + eps
    return p + (-(lr / (1.0 - beta1 ** t))) * (m / den), m, v


def resnet18_tensors():
    """(name, shape KRSC or [C], input H) of the 62 trainable tensors of torchvision's ResNet-18 (11,689,512 elements): conv filters
    with the spatial size of their input, BN gamma / beta with H 0, the fc weight [1000][1][1][512] and its bias"""
    out = [("conv1", (64, 7, 7, 3), 224), ("bn1.g", (64,), 0), ("bn1.b", (64,), 0)]
    cin, h = 64, 56
    for li, cout in enumerate((64, 128, 256, 512), 1):
        for bi in range(2):
            stride = 2 if li > 1 and bi == 0 else 1
            c0 = cin if bi == 0 else cout
            out += [(f"layer{li}.{bi}.conv1", (cout, 3, 3, c0), h), (f"layer{li}.{bi}.bn1.g", (cout,), 0), (f"layer{li}.{bi}.bn1.b", (cout,), 0)]
            h2 = h // stride
            out += [(f"layer{li}.{bi}.conv2", (cout, 3, 3, cout), h2), (f"layer{li}.{bi}.bn2.g", (cout,), 0), (f"layer{li}.{bi}.bn2.b", (cout,), 0)]
            if stride == 2:
                out += [(f"layer{li}.{bi}.down", (cout, 1, 1, c0), h), (f"layer{li}.{bi}.downbn.g", (cout,), 0),
                        (f"layer{li}.{bi}.downbn.b", (cout,), 0)]
            h = h2
        cin = cout
    return out + [("fc.w", (1000, 1, 1, 512), 0), ("fc.b", (1000,), 0)]
