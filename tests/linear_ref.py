"""float64 references of the fully connected layer (pcnn_linear_plan_create / _wgrad / _dgrad) and of the bf16 softmax
cross-entropy (pcnn_softmax_ce_bf16).  test_linear_cpu.py pins them to torch.nn.functional.linear, cross_entropy and autograd.

Shapes: x [N][P][Q][C] (NHWC, flattened to F = P*Q*C features in that order), w [O][P][Q][C], b [O], y and dy [N][O]."""
import numpy as np


def flat(a):
    return np.asarray(a, np.float64).reshape(a.shape[0], -1)


def fwd_f64(x, w, b=None, act=0):
    """act(x w^T + b) in float64"""
    pre = flat(x) @ flat(w).T
    if b is not None:
        pre = pre + np.asarray(b, np.float64)
    return 1.0 / (1.0 + np.exp(-pre)) if act else pre


def wgrad_f64(x, dy):
    """dW [O][P][Q][C] = dy^T x"""
    return (np.asarray(dy, np.float64).T @ flat(x)).reshape((dy.shape[1],) + tuple(x.shape[1:]))


def dgrad_f64(dy, w):
    """dx [N][P][Q][C] = dy w"""
    return (np.asarray(dy, np.float64) @ flat(w)).reshape((dy.shape[0],) + tuple(w.shape[1:]))


def softmax_ce_f64(z, labels, scale):
    """(g, loss, pred): g = (softmax(z) - onehot(label)) * scale, loss = -log p_label, pred = the first index of the largest
    logit, evaluated as pcnn_softmax_ce_bf16 documents (max-shifted, in float64).  A row holding NaN: g and loss NaN, pred -1.
    A label >= O: g and loss NaN, pred the argmax."""
    z = np.asarray(z, np.float64)
    labels = np.asarray(labels).astype(np.int64)
    N, O = z.shape
    rows = np.arange(N)
    m = z.max(axis=1, keepdims=True)
    e = np.exp(z - m)
    den = e.sum(axis=1, keepdims=True)
    valid = labels < O
    onehot = np.zeros_like(z)
    onehot[rows[valid], labels[valid]] = 1.0
    with np.errstate(invalid="ignore"):
        g = (e / den - onehot) * scale
        loss = -((z[rows, np.minimum(labels, O - 1)] - m[:, 0]) - np.log(den[:, 0]))
    nan = np.isnan(z).any(axis=1)
    bad = nan | ~valid
    g[bad] = np.nan
    loss[bad] = np.nan
    pred = np.where(nan, -1, np.argmax(np.where(np.isnan(z), -np.inf, z), axis=1))
    return g, loss, pred


def f64_to_bf16_bits(pkg, g):
    """the documented rounding of dlogits: float64 -> fp32 -> bf16, each to nearest even"""
    return pkg.f32_to_bf16_bits(np.asarray(g, np.float64).astype(np.float32))


def near_boundary(pkg, g, rel=1e-12):
    """elements whose float64 -> fp32 -> bf16 result changes within a relative 1e-12 of g: the device's exp and summation order
    may land on either side, so one bf16 ulp is allowed there"""
    lo = f64_to_bf16_bits(pkg, np.asarray(g) * (1 - rel))
    hi = f64_to_bf16_bits(pkg, np.asarray(g) * (1 + rel))
    return lo != hi
