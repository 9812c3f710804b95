"""numpy replays of the squeeze-and-excitation channel scale (pcnn_se_scale_nhwc_bf16_fwd / _bwd_gate / _bwd_input, include/pcnn.h)
on arrays [N][H][W][C] with the gate s and its gradient ds [N][C] and the squeeze branch's gradient dpool [N][C], and float64
references, including the whole block: GAP -> fc1 + ReLU -> fc2 + sigmoid -> scale.

In float32 every operation below is the kernels' own, in their order: numpy multiplies, adds and divides float32 arrays with one
IEEE rounding each.  bf16 values are carried as float32 arrays; bf16() rounds to nearest even as the kernels do (NaN stays NaN)."""
import numpy as np


def bf16(a):
    """float32 -> the nearest bf16 value (ties to even) as float32; NaN -> NaN"""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    r = (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32)
    return np.where(nan, np.float32(np.nan), r.view(np.float32))


def relu(v):
    """v < 0 ? +0 : v, NaN and -0 unchanged"""
    return np.where(v < 0, np.zeros((), v.dtype), v)


def fwd(x, s, r=None, act=0):
    """y before the bf16 rounding, in x's dtype: act(x * s (+ r))"""
    with np.errstate(all="ignore"):
        v = x * s[:, None, None, :]
        if r is not None:
            v = v + r
    return relu(v) if act == 3 else v


def gate_g(dy, y=None, dy2=None, act=0):
    """g (bf16 values as float32): dy, or bf16(dy + dy2); +0 where y <= 0 at act 3 (a NaN y passes)"""
    with np.errstate(all="ignore"):
        g = dy.copy() if dy2 is None else bf16(dy + dy2)
    if act == 3:
        g = np.where(y <= 0, np.float32(0), g)
    return g


def ordered_sum(p, info):
    """the sum over the pixels of p [N][H][W][C] (float32) in the partition `info` (se_scale_nhwc_info): in each range of
    pixels_per_cta pixels, lane l sums the pixels l, l + lanes, ... from its first; the lanes holding a pixel are added in lane
    order, then the ranges in range order"""
    N, H, W, C = p.shape
    HW = H * W
    ps = p.reshape(N, HW, C)
    lanes, per = info["lanes"], info["pixels_per_cta"]
    assert info["ranges"] == -(-HW // per)
    total = None
    with np.errstate(all="ignore"):
        for p0 in range(0, HW, per):
            acc = np.full((N, lanes, C), -0.0, np.float32)
            for j in range(per // lanes):
                px = p0 + j * lanes + np.arange(lanes)
                ok = px < HW
                acc[:, ok] = acc[:, ok] + ps[:, px[ok]]
            s = acc[:, 0]
            for lane in range(1, min(lanes, HW - p0)):
                s = s + acc[:, lane]
            total = s if total is None else total + s
    return total


def gate_ds(g, x, info):
    """ds before the bf16 rounding: the ordered float32 sum of g * x"""
    with np.errstate(all="ignore"):
        return ordered_sum(g * x, info)


def dx(g, s, dpool=None, HW=1):
    """dx before the bf16 rounding, in g's dtype: g * s (+ dpool / HW)"""
    with np.errstate(all="ignore"):
        v = g * s[:, None, None, :]
        if dpool is not None:
            v = v + (dpool / g.dtype.type(HW))[:, None, None, :]
    return v


def sigmoid_bwd(ds, s):
    """pcnn_conv_bias_act_bwd at act 1 before the bf16 rounding: ds * (s * (1 - s))"""
    with np.errstate(all="ignore"):
        return ds * (s * (np.float32(1) - s))


# ------------------------------------------------------------------ float64: the scale and the whole block
def gate64(x, dy, y=None, dy2=None, act=0):
    """(g, ds) in float64: g = act'(dy + dy2) (y <= 0 gives 0 at act 3), ds = the sum over the pixels of g * x"""
    t = dy if dy2 is None else dy + dy2
    g = np.where(y <= 0, 0.0, t) if act == 3 else t
    return g, (g * x).sum(axis=(1, 2))


def block_fwd64(x, w1, b1, w2, b2, r=None, act=0):
    """the SE block in float64: h = mean over the pixels, a = relu(h w1^T + b1), s = sigmoid(a w2^T + b2), y = act(x s + r)"""
    h = x.mean(axis=(1, 2))
    a = np.maximum(h @ w1.T + b1, 0.0)
    s = 1.0 / (1.0 + np.exp(-(a @ w2.T + b2)))
    return dict(h=h, a=a, s=s, y=fwd(x, s, r, act))


def block_bwd64(x, f, w1, w2, dy, dy2=None, act=0):
    """the SE block's backward in float64 in the layer's order: the gate pass, fc2's backward (sigmoid), fc1's backward (ReLU),
    the input pass with dpool = fc1's dx.  f is block_fwd64's dict.  Returns g (= dr), dx, and the four parameter gradients."""
    N, H, W, C = x.shape
    g, ds = gate64(x, dy, f["y"], dy2, act)
    d2 = ds * f["s"] * (1.0 - f["s"])
    dw2, db2, da = d2.T @ f["a"], d2.sum(0), d2 @ w2
    d1 = np.where(f["a"] > 0, da, 0.0)
    dw1, db1, dh = d1.T @ f["h"], d1.sum(0), d1 @ w1
    return dict(g=g, ds=ds, dx=dx(g, f["s"], dh, H * W), dw1=dw1, db1=db1, dw2=dw2, db2=db2)
