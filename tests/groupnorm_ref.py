"""References of group normalization with a fused residual add and activation (pcnn_groupnorm_nhwc_bf16_fwd / _bwd /
_bwd_preact), on dense [N][HW][C] arrays with G groups of Cg = C / G channels:

- float64: fwd_f64 / bwd_f64, which test_groupnorm_cpu.py pins to torch.nn.functional.group_norm and its autograd (and, at G = C
  and G = 1, to instance_norm and layer_norm), with the add and every activation code;
- numpy float32 replays of the formulas of include/pcnn.h given the statistics and the group sums the device computed: fwd_bits
  (y), grad_bits (g, which is also dr) and dx_bits.  The per-element rules are batch normalization's with the group's statistics,
  so these call batchnorm_ref's and bnact_ref's replays on statistics expanded to channels.

numpy float32 arithmetic is IEEE round to nearest with no contraction, which is what the kernels use.  check_stats and
check_sums state the error model of the device's statistics and sums: fp32 partials of at most n_acc roundings each (the info
query's n_acc and n_acc_group), merged in double."""
import numpy as np

import batchnorm_ref as BR
import bnact_ref as BA

F32 = np.float32
U = 2.0 ** -24


def per_channel(stat, C):
    """[N][G] -> [N][1][C]: each channel's entry of its group"""
    stat = np.asarray(stat).reshape(stat.shape[0], -1)
    return np.repeat(stat, C // stat.shape[1], axis=1)[:, None, :]


def group_view(a, G):
    """[N][HW][C] -> [N][G][HW * Cg]: the elements of each (image, group)"""
    N, HW, C = a.shape
    return np.asarray(a).reshape(N, HW, G, C // G).transpose(0, 2, 1, 3).reshape(N, G, -1)


def act_f64(v, act):
    if act == 0:
        return v
    if act == 3:
        return BR.relu(v)
    return BA.act_f64(v, act)


# ------------------------------------------------------------------------------------------------ float64
def fwd_f64(x, gamma, beta, G, r=None, act=0, eps=1e-5):
    """y = act((x - mean) / sqrt(var + eps) * gamma + beta (+ r)) over [N][HW][C], mean and the biased var of each (n, g); returns
    y, the pre-activation v, mean [N][G] and var [N][G]"""
    x = np.asarray(x, np.float64)
    C = x.shape[2]
    xg = group_view(x, G)
    mean, var = xg.mean(axis=2), xg.var(axis=2)
    xhat = (x - per_channel(mean, C)) / np.sqrt(per_channel(var, C) + eps)
    v = xhat * np.asarray(gamma, np.float64) + np.asarray(beta, np.float64)
    if r is not None:
        v = v + np.asarray(r, np.float64)
    with np.errstate(all="ignore"):
        return act_f64(v, act), v, mean, var


def bwd_f64(x, gamma, beta, G, dy, dy2=None, r=None, act=0, eps=1e-5):
    """Gradients of the forward above: dx, dgamma, dbeta, g (the gradient of v and of r), and A, B [N][G] = the group sums of
    gamma * g and gamma * g * xhat"""
    x = np.asarray(x, np.float64)
    N, HW, C = x.shape
    _, v, mean, var = fwd_f64(x, gamma, beta, G, r, 0, eps)
    t = np.asarray(dy, np.float64) + (0 if dy2 is None else np.asarray(dy2, np.float64))
    with np.errstate(all="ignore"):
        g = t if act == 0 else np.where(v <= 0, 0.0, t) if act == 3 else BA.dact_f64(v, t, act)
    rstd = 1 / np.sqrt(per_channel(var, C) + eps)
    xhat = (x - per_channel(mean, C)) * rstd
    ga = np.asarray(gamma, np.float64)
    dbeta, dgamma = g.sum(axis=(0, 1)), (g * xhat).sum(axis=(0, 1))
    A, B = group_view(ga * g, G).sum(axis=2), group_view(ga * g * xhat, G).sum(axis=2)
    Mg = HW * (C // G)
    dx = ((ga * g - per_channel(A, C) / Mg) - xhat * per_channel(B, C) / Mg) * rstd
    return dx, dgamma, dbeta, g, A, B


# ------------------------------------------------------------------------------------------------ float32 replays
def xhat32(pkg, x_bits, mean, rstd):
    C = x_bits.shape[2]
    return BR.xhat32(pkg, x_bits, per_channel(np.asarray(mean, F32), C), per_channel(np.asarray(rstd, F32), C))


def pre32(pkg, x_bits, gamma, beta, mean, rstd, r_bits=None):
    """v = RN(RN(xhat gamma) + beta) (+ float(r)) with each element's group statistics"""
    C = x_bits.shape[2]
    return BA.pre32(pkg, x_bits, gamma, beta, per_channel(np.asarray(mean, F32), C), per_channel(np.asarray(rstd, F32), C), r_bits)


def fwd_bits(pkg, x_bits, gamma, beta, mean, rstd, r_bits=None, act=0):
    """y bits: bf16_rn(act(v)), act as in batch normalization's forward"""
    v = pre32(pkg, x_bits, gamma, beta, mean, rstd, r_bits)
    if act in BA.CODES:
        return BA.act_bits(pkg, v, act)
    return pkg.f32_to_bf16_bits(BR.relu(v) if act == 3 else v)


def grad_bits(pkg, x_bits, gamma, beta, mean, rstd, dy_bits, dy2_bits=None, r_bits=None, act=0, y_bits=None):
    """g bits: from y at codes 0 and 3 (batchnorm_ref.grad_bits), from the recomputed pre-activation at 4-6 (bnact_ref.grad_bits)"""
    if act in BA.CODES:
        return BA.grad_bits(pkg, pre32(pkg, x_bits, gamma, beta, mean, rstd, r_bits), dy_bits, dy2_bits, act)
    return BR.grad_bits(pkg, y_bits, dy_bits, dy2_bits, act)


def dx_bits(pkg, x_bits, g_bits, gamma, mean, rstd, dstat):
    """dx bits: bf16_rn(RN(RN(RN(RN(g gamma) - a) - RN(xhat b)) rstd)), a = RN(A / Mgf), b = RN(B / Mgf), Mgf = float(HW Cg)"""
    N, HW, C = x_bits.shape
    dstat = np.asarray(dstat, F32).reshape(2, N, -1)
    Mgf = F32(HW * (C // dstat.shape[2]))
    a, b = per_channel(dstat[0] / Mgf, C), per_channel(dstat[1] / Mgf, C)
    t = ((pkg.bf16_bits_to_f32(g_bits) * np.asarray(gamma, F32)) - a) - xhat32(pkg, x_bits, mean, rstd) * b
    return pkg.f32_to_bf16_bits(t * per_channel(np.asarray(rstd, F32), C))


# ------------------------------------------------------------------------------------------------ error model
def check_stats(pkg, xb, G, mean, rstd, eps, n):
    """the device's group means and variances (read back from rstd) within the error model of float64 over x's bf16 bits:
    |mean - m64| <= n u R + u |m64| and |var - v64| <= 5 n u R^2 + 4 u (v64 + eps), R the group's range, n = n_acc_group"""
    xg = group_view(pkg.bf16_bits_to_f32(xb).astype(np.float64), G)
    m64, v64 = xg.mean(axis=2), xg.var(axis=2)
    R = xg.max(axis=2) - xg.min(axis=2)
    mean, rstd = np.asarray(mean, np.float64).reshape(m64.shape), np.asarray(rstd, np.float64).reshape(m64.shape)
    var = 1.0 / rstd ** 2 - np.float64(F32(eps))
    assert np.all(np.abs(mean - m64) <= n * U * R + U * np.abs(m64)), np.abs(mean - m64).max()
    bound = 5 * n * U * R ** 2 + 4 * U * (v64 + eps)
    assert np.all(np.abs(var - v64) <= bound), (np.abs(var - v64) / bound).max()


def sums64(pkg, x_bits, g_bits, gamma, mean, rstd, G):
    """float64 sums of the device's fp32 terms: dbeta, dgamma [C] and A, B [N][G], with the Sigma |terms| of each"""
    g = pkg.bf16_bits_to_f32(g_bits).astype(np.float64)
    gx = g * xhat32(pkg, x_bits, mean, rstd).astype(np.float64)
    ga = np.asarray(gamma, F32).astype(np.float64)
    out = {"dbeta": (g.sum(axis=(0, 1)), np.abs(g).sum(axis=(0, 1))), "dgamma": (gx.sum(axis=(0, 1)), np.abs(gx).sum(axis=(0, 1))),
           "A": (group_view(ga * g, G).sum(axis=2), group_view(np.abs(ga * g), G).sum(axis=2)),
           "B": (group_view(ga * gx, G).sum(axis=2), group_view(np.abs(ga * gx), G).sum(axis=2))}
    return out


def check_sums(pkg, x_bits, g_bits, gamma, mean, rstd, G, dgamma, dbeta, dstat, info):
    """dgamma, dbeta within 2 n_acc u Sigma |terms| of float64, A and B within 2 n_acc_group u Sigma |terms|; returns the worst
    ratio to the bound of each"""
    N = x_bits.shape[0]
    ref = sums64(pkg, x_bits, g_bits, gamma, mean, rstd, G)
    dstat = np.asarray(dstat, np.float64).reshape(2, N, G)
    got = {"dbeta": np.asarray(dbeta, np.float64), "dgamma": np.asarray(dgamma, np.float64), "A": dstat[0], "B": dstat[1]}
    worst = {}
    for k, (v64, mag) in ref.items():
        n = info["n_acc"] if k in ("dbeta", "dgamma") else info["n_acc_group"]
        bound = 2 * n * U * mag
        err = np.abs(got[k] - v64)
        assert np.all(err <= bound), (k, (err / np.maximum(bound, 1e-300)).max())
        worst[k] = float((err / np.maximum(bound, 1e-300)).max())
    return worst
