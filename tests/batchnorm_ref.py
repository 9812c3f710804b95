"""References of batch normalization with a fused residual add and ReLU (pcnn_batchnorm_nhwc_bf16_fwd / _bwd), on dense
[pixels][C] arrays:

- float64: fwd_f64 / bwd_f64, which test_batchnorm_cpu.py pins to torch.nn.functional.batch_norm (training and eval, running
  statistics included) and to its autograd, with the add and the ReLU;
- numpy float32 replays of the formulas of include/pcnn.h, every operation rounded as the kernels round it, given the statistics,
  dgamma and dbeta the device computed: fwd_bits, eval_rstd, running_update, grad_bits and dx_bits.

numpy float32 arithmetic is IEEE round to nearest with no contraction, which is what the kernels use.

n_stat, n_acc and check_stats state the error model of the device's statistics and gradient sums (test_batchnorm_gpu.py's
docstring derives it)."""
import numpy as np

F32 = np.float32
U = 2.0 ** -24
ITERS = 16


def n_stat(pkg, pixels, C):
    return ITERS + pkg.batchnorm_nhwc_info(pixels, C)["lanes"] + 3


def n_acc(pkg, pixels, C):
    info = pkg.batchnorm_nhwc_info(pixels, C)
    return ITERS + info["lanes"] + -(-info["grad_slots"] // 8) + 3


def check_stats(pkg, xb, mean, rstd, eps):
    """the device's batch mean and variance (read back from rstd) within the error model of float64 over x's bf16 bits [pixels][C];
    returns the float64 mean, variance and the variance bound"""
    pixels, C = xb.shape
    x = pkg.bf16_bits_to_f32(xb).astype(np.float64)
    m64, v64 = x.mean(0), ((x - x.mean(0)) ** 2).mean(0)
    R = x.max(0) - x.min(0)
    n = n_stat(pkg, pixels, C)
    var = 1.0 / rstd.astype(np.float64) ** 2 - np.float64(np.float32(eps))
    assert np.all(np.abs(mean - m64) <= n * U * R + U * np.abs(m64)), np.abs(mean - m64).max()
    bound = 5 * n * U * R ** 2 + 4 * U * (v64 + eps)
    assert np.all(np.abs(var - v64) <= bound), (np.abs(var - v64) / bound).max()
    return m64, v64, bound


def relu(v):
    v = np.asarray(v)
    return np.where(v < 0, np.zeros((), v.dtype), v)


# ------------------------------------------------------------------------------------------------ float64
def fwd_f64(x, gamma, beta, r=None, act=0, training=True, eps=1e-5, momentum=0.1, running_mean=None, running_var=None):
    """y = act((x - mean) / sqrt(var + eps) * gamma + beta (+ r)) over [M][C]; returns y, mean, biased var and the updated running
    statistics (None where not given).  eval uses the running statistics and leaves them."""
    x = np.asarray(x, np.float64)
    M = x.shape[0]
    rm = None if running_mean is None else np.asarray(running_mean, np.float64)
    rv = None if running_var is None else np.asarray(running_var, np.float64)
    if training:
        mean = x.mean(axis=0)
        var = ((x - mean) ** 2).mean(axis=0)
        if rm is not None:
            rm = (1 - momentum) * rm + momentum * mean
            rv = (1 - momentum) * rv + momentum * var * M / (M - 1)
    else:
        mean, var = rm, rv
    v = (x - mean) / np.sqrt(var + eps) * np.asarray(gamma, np.float64) + np.asarray(beta, np.float64)
    if r is not None:
        v = v + np.asarray(r, np.float64)
    return (relu(v) if act == 3 else v), mean, var, rm, rv


def bwd_f64(x, gamma, y, dy, dy2=None, act=0, eps=1e-5):
    """Gradients of a training forward whose output was y: dx, dgamma, dbeta and dr (the gradient of r)"""
    x = np.asarray(x, np.float64)
    M = x.shape[0]
    t = np.asarray(dy, np.float64) + (0 if dy2 is None else np.asarray(dy2, np.float64))
    g = np.where(np.asarray(y) <= 0, 0.0, t) if act == 3 else t
    mean = x.mean(axis=0)
    rstd = 1 / np.sqrt(((x - mean) ** 2).mean(axis=0) + eps)
    xhat = (x - mean) * rstd
    dbeta, dgamma = g.sum(axis=0), (g * xhat).sum(axis=0)
    dx = (g - dbeta / M - xhat * (dgamma / M)) * (np.asarray(gamma, np.float64) * rstd)
    return dx, dgamma, dbeta, g


# ------------------------------------------------------------------------------------------------ float32 replays
def xhat32(pkg, x_bits, mean, rstd):
    return (pkg.bf16_bits_to_f32(x_bits) - np.asarray(mean, F32)) * np.asarray(rstd, F32)


def fwd_bits(pkg, x_bits, gamma, beta, mean, rstd, r_bits=None, act=0):
    """y bits: bf16_rn(act((float(x) - mean) * rstd * gamma + beta (+ float(r)))), fp32 in this order"""
    v = xhat32(pkg, x_bits, mean, rstd) * np.asarray(gamma, F32) + np.asarray(beta, F32)
    if r_bits is not None:
        v = v + pkg.bf16_bits_to_f32(r_bits)
    return pkg.f32_to_bf16_bits(relu(v) if act == 3 else v)


def eval_rstd(running_var, eps):
    """float(1 / sqrt(double(running_var) + double(eps)))"""
    return (1.0 / np.sqrt(np.asarray(running_var, F32).astype(np.float64) + np.float64(F32(eps)))).astype(F32)


def running_update(running, stat, momentum):
    """keep * running + momentum * stat in fp32, keep = 1 - momentum in fp32"""
    m = F32(momentum)
    return (F32(1) - m) * np.asarray(running, F32) + m * np.asarray(stat, F32)


def grad_bits(pkg, y_bits, dy_bits, dy2_bits=None, act=0):
    """g~ bits: bf16_rn(act'(float(dy) (+ float(dy2)))); without dy2 dy's bits pass; at act 3 float(y) <= 0 gives +0"""
    if dy2_bits is None:
        g = np.asarray(dy_bits, np.uint16).copy()
    else:
        g = pkg.f32_to_bf16_bits(pkg.bf16_bits_to_f32(dy_bits) + pkg.bf16_bits_to_f32(dy2_bits))
    if act == 3:
        with np.errstate(invalid="ignore"):
            g = np.where(pkg.bf16_bits_to_f32(y_bits) <= 0, np.uint16(0), g).astype(np.uint16)
    return g


def dx_bits(pkg, x_bits, g_bits, gamma, mean, rstd, dgamma, dbeta):
    """dx bits: bf16_rn(((g - dbeta / Mf) - xhat * (dgamma / Mf)) * (gamma * rstd)), Mf = float(M)"""
    Mf = F32(x_bits.shape[0])
    mb, mg = np.asarray(dbeta, F32) / Mf, np.asarray(dgamma, F32) / Mf
    sc = np.asarray(gamma, F32) * np.asarray(rstd, F32)
    t = (pkg.bf16_bits_to_f32(g_bits) - mb) - xhat32(pkg, x_bits, mean, rstd) * mg
    return pkg.f32_to_bf16_bits(t * sc)
