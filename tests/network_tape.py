"""A tape of one network's real run on the device, and one host checker per tape entry (TEST INFRASTRUCTURE ONLY).

Tape(eng, net) wraps the bound methods of one network instance: every layer's forward and backward (the pools' and the global
pool's included) and the engine's softmax_ce_bf16.  The network class's own forward and backward then run unchanged.  Each wrapper
synchronises and snapshots everything the call reads (its buffer arguments, the layer's kept _x in a backward, the fp32 masters and
the batch-norm statistics as they are at that moment), runs the call, synchronises again and snapshots everything the call wrote.
A dy that a layer with an activation rewrites in place is snapshotted before and after.  A buffer passed as a raw device pointer
(the stem's x, a pointer into the MNIST tensor) is read from the tensor registered for it in Tape.inputs.

check(pkg, entry, full) compares one call with float64 (or with a float32 replay, bit for bit) on the operands the call was
actually given, with the bounds the per-layer tests justify.  Weights always come from the master read back at the time of the
call, rounded to bf16: a plan whose bf16 operands went stale fails.  full=False runs only the bit-exact checks and the batch
statistics (a training batch-norm forward stores its float64 variance and bound in entry["stats"]).  Each check asserts and
returns {check name: worst ratio to its bound} (0 for a bit-exact check, which fails on any difference)."""
import inspect

import numpy as np
import torch

import avgpool_ref as AR
import batchnorm_ref as BR
import conv_ref as CR
import conv_ref_strided as CS
import dwconv_ref as DR
import linear_ref as LR
import maxpool_ref as MR
import relu_ref as RR

U = 2.0 ** -24
BUFFERS = {"x", "y", "dy", "dx", "r", "dr", "dy2", "logits", "labels", "dlogits", "loss", "pred"}
OUTPUTS = {"forward": {"y"}, "backward": {"dx", "dr"}, "softmax": {"dlogits", "loss", "pred"}}
# (class name, op) -> layer attributes read before the call and written by it
STATE_IN = {("ConvLayer", "forward"): ("filt", "bias"), ("ConvLayer", "backward"): ("filt", "bias", "_x"),
            ("DepthwiseConvLayer", "forward"): ("filt", "bias"), ("DepthwiseConvLayer", "backward"): ("filt", "bias", "_x"),
            ("LinearLayer", "forward"): ("w", "bias"), ("LinearLayer", "backward"): ("w", "bias", "_x"),
            ("BatchNormLayer", "forward"): ("gamma", "beta", "running_mean", "running_var"),
            ("BatchNormLayer", "backward"): ("gamma", "save_mean", "save_rstd", "_x"),
            ("MaxPoolLayer", "backward"): ("argmax",)}
STATE_OUT = {("ConvLayer", "backward"): ("dw", "db"), ("DepthwiseConvLayer", "backward"): ("dw", "db"),
             ("LinearLayer", "backward"): ("dw", "db"),
             ("BatchNormLayer", "forward"): ("save_mean", "save_rstd", "running_mean", "running_var"),
             ("BatchNormLayer", "backward"): ("dgamma", "dbeta"), ("MaxPoolLayer", "forward"): ("argmax",)}
KINDS = ("ConvLayer", "DepthwiseConvLayer", "LinearLayer", "BatchNormLayer", "MaxPoolLayer", "AvgPoolLayer", "GlobalAvgPoolLayer")


def layers_of(net):
    """(name, layer) of every layer object the network holds, as attributes or in lists of attributes"""
    out = []
    for k, v in vars(net).items():
        for i, item in enumerate(v if isinstance(v, (list, tuple)) else [v]):
            if type(item).__name__ in KINDS:
                out.append((f"{k}[{i}]" if isinstance(v, (list, tuple)) else k, item))
    return out


class Tape:
    """with Tape(eng, net) as tape: ... records every call into tape.sink(entry) (default: tape.entries.append); tape.step is
    stored in each entry.  Leaving the block restores the network's and the engine's own methods."""

    def __init__(self, eng, net):
        self.eng, self.net = eng, net
        self.inputs = {}
        self.entries = []
        self.sink = self.entries.append
        self.step = None
        self._undo = []

    def __enter__(self):
        for name, layer in layers_of(self.net):
            for op in ("forward", "backward"):
                self._wrap(layer, op, name, type(layer).__name__)
        self._wrap(self.eng, "softmax_ce_bf16", "softmax", "softmax")
        return self

    def __exit__(self, *exc):
        for obj, op in self._undo:
            delattr(obj, op)
        self._undo = []

    def snap(self, a):
        if a is None:
            return None
        if isinstance(a, int):
            a = self.inputs[a]
        if isinstance(a, torch.Tensor):
            h = a.detach().cpu().numpy().copy()
            return h.view(np.uint16) if h.dtype == np.int16 else h
        return a.to_host()

    def _wrap(self, obj, op, name, kind):
        orig = getattr(obj, op)
        sig = inspect.signature(orig)
        kop = "softmax" if kind == "softmax" else op

        def call(*args, **kw):
            bound = sig.bind(*args, **kw)
            bound.apply_defaults()
            argv = dict(bound.arguments)
            self.eng.sync()
            a = {k: self.snap(v) for k, v in argv.items() if k in BUFFERS and k not in OUTPUTS[kop]}
            for attr in STATE_IN.get((kind, op), ()):
                a[attr] = self.snap(getattr(obj, attr))
            out = orig(*args, **kw)
            self.eng.sync()
            o = {k: self.snap(argv[k]) for k in OUTPUTS[kop] if k in argv}
            if op == "backward" and "dy" in argv:
                o["dy"] = self.snap(argv["dy"])
            for attr in STATE_OUT.get((kind, op), ()):
                o[attr] = self.snap(getattr(obj, attr))
            self.sink(dict(step=self.step, name=name, kind=kind, op=kop, layer=obj, argv=argv, a=a, o=o))
            return out

        setattr(obj, op, call)
        self._undo.append((obj, op))


# ------------------------------------------------------------------------------------------------ checkers
def _ratio(err, bound):
    r = float(np.max(np.abs(err) / (bound + 1e-30)))
    assert r <= 1.0, r
    return r


def _exact(got, want, what):
    bad = int(np.sum(np.asarray(got) != np.asarray(want)))
    assert bad == 0, f"{what}: {bad} elements differ"
    return 0.0


def _positive(pkg, y, what):
    frac = float((pkg.bf16_bits_to_f32(y) > 0).mean())
    assert 0.05 < frac < 0.95, f"{what}: {frac:.3f} of the ReLU outputs are positive"
    return frac


def _img(bits, N, rows, pitch, h, wc):
    """the h x wc image of a [N][rows][pitch] buffer"""
    return bits.reshape(N, rows, pitch)[:, :h, :wc]


def _bfw(pkg, w):
    return pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(w)).astype(np.float64)


def _act_ref(pre, acc, act):
    """float64 reference of an epilogue and its bound: the fp32 accumulation bound acc plus one bf16 rounding of y; the sigmoid's
    tanh.approx adds 1e-3"""
    if act == 1:
        ref = 1 / (1 + np.exp(-pre))
        return ref, acc / 4 + 2.0 ** -8 * np.abs(ref) + 1e-3
    if act == 3:
        ref = RR.relu(pre)
        return ref, acc + 2.0 ** -8 * ref
    return pre, acc + 2.0 ** -8 * np.abs(pre)


def _dpre(pkg, e, act, what):
    """dy rewritten in place by the bias / activation backward: bit-identical to the replay on y and the dy given"""
    y, dy0, dy1 = e["a"]["y"], e["a"]["dy"], e["o"]["dy"]
    if act == 3:
        want = RR.bwd_bits(pkg, y, dy0)
    elif act == 1:
        y32 = pkg.bf16_bits_to_f32(y)
        want = pkg.f32_to_bf16_bits(pkg.bf16_bits_to_f32(dy0) * (y32 * (np.float32(1) - y32)))
    else:
        want = dy0
    return _exact(dy1, want, what + " dpre")


def conv_forward(pkg, e, full):
    L, a = e["layer"], e["a"]
    N, H, W, C, K, R, S = L.shape
    (ph, pw), st = L.padding, L.stride
    y = e["o"]["y"].reshape(L.out_shape)
    r = {}
    if L.act == 3:
        _positive(pkg, y, e["name"])
    if not full:
        return r
    x = pkg.bf16_bits_to_f32(_img(a["x"], N, L.image_rows or H, L.row_pitch, H, W * C)).astype(np.float64).reshape(N, H, W, C)
    w, b = _bfw(pkg, a["filt"]), a["bias"]
    xp = np.pad(x, ((0, 0), (ph, ph), (pw, pw), (0, 0)))
    pre = CR.conv_fwd_f64(xp, w, b, st)
    acc = 2 * R * S * C * U * CR.conv_fwd_f64(np.abs(xp), np.abs(w), None if b is None else np.abs(b), st)
    ref, bound = _act_ref(pre, acc, L.act)
    r["y"] = _ratio(pkg.bf16_bits_to_f32(y) - ref, bound)
    return r


def conv_backward(pkg, e, full):
    L, a, o = e["layer"], e["a"], e["o"]
    N, H, W, C, K, R, S = L.shape
    (ph, pw), st = L.padding, L.stride
    r = {"dpre": _dpre(pkg, e, L.act, e["name"])}
    if not full:
        return r
    x = pkg.bf16_bits_to_f32(_img(a["_x"], N, L.image_rows or H, L.row_pitch, H, W * C)).astype(np.float64).reshape(N, H, W, C)
    xp = np.pad(x, ((0, 0), (ph, ph), (pw, pw), (0, 0)))
    d = pkg.bf16_bits_to_f32(o["dy"]).astype(np.float64).reshape(L.out_shape)
    n = L.pixels
    r["dw"] = _ratio(o["dw"] - CS.conv_wgrad_f64(xp, d, R, S, st), 2 * n * U * CS.conv_wgrad_f64(np.abs(xp), np.abs(d), R, S, st))
    if o["db"] is not None:
        r["db"] = _ratio(o["db"] - d.sum(axis=(0, 1, 2)), 2 * n * U * np.abs(d).sum(axis=(0, 1, 2)))
    if o.get("dx") is not None:
        w = _bfw(pkg, a["filt"])
        crop = lambda v: v[:, ph:ph + H, pw:pw + W, :]
        ref = crop(CS.conv_dgrad_f64(d, w, H + 2 * ph, W + 2 * pw, st))
        acc = crop(CS.conv_dgrad_f64(np.abs(d), np.abs(w), H + 2 * ph, W + 2 * pw, st))
        got = pkg.bf16_bits_to_f32(_img(o["dx"], N, L.image_rows or H, L.row_pitch, H, W * C)).reshape(N, H, W, C)
        r["dx"] = _ratio(got - ref, 2.0 ** -8 * np.abs(ref) + 2 * K * R * S * U * acc)
    return r


def linear_forward(pkg, e, full):
    L, a = e["layer"], e["a"]
    N, P, Q, C, O = L.shape
    y = e["o"]["y"].reshape(N, O)
    r = {}
    if L.act == 3:
        _positive(pkg, y, e["name"])
    if not full:
        return r
    x = pkg.bf16_bits_to_f32(_img(a["x"], N, L.image_rows or P, L.row_pitch, P, Q * C)).astype(np.float64).reshape(N, P, Q, C)
    w = _bfw(pkg, a["w"])
    pre = LR.fwd_f64(x, w, a["bias"])
    ref, bound = _act_ref(pre, 2 * P * Q * C * U * LR.fwd_f64(np.abs(x), np.abs(w)), L.act)
    r["y"] = _ratio(pkg.bf16_bits_to_f32(y) - ref, bound)
    return r


def linear_backward(pkg, e, full):
    L, a, o = e["layer"], e["a"], e["o"]
    N, P, Q, C, O = L.shape
    r = {"dpre": _dpre(pkg, e, L.act, e["name"])}
    if not full:
        return r
    x = pkg.bf16_bits_to_f32(_img(a["_x"], N, L.image_rows or P, L.row_pitch, P, Q * C)).astype(np.float64).reshape(N, P, Q, C)
    d = pkg.bf16_bits_to_f32(o["dy"]).astype(np.float64).reshape(N, O)
    r["dw"] = _ratio(o["dw"] - LR.wgrad_f64(x, d), 2 * N * U * LR.wgrad_f64(np.abs(x), np.abs(d)))
    if o["db"] is not None:
        r["db"] = _ratio(o["db"] - d.sum(0), 2 * N * U * np.abs(d).sum(0))
    if o.get("dx") is not None:
        w = _bfw(pkg, a["w"])
        ref, acc = LR.dgrad_f64(d, w), LR.dgrad_f64(np.abs(d), np.abs(w))
        got = pkg.bf16_bits_to_f32(_img(o["dx"], N, L.image_rows or P, L.row_pitch, P, Q * C)).reshape(N, P, Q, C)
        r["dx"] = _ratio(got - ref, 2 * O * U * acc + 2.0 ** -8 * np.abs(ref))
    return r


def dwconv_forward(pkg, e, full):
    L, a = e["layer"], e["a"]
    N, H, W, C, R, S = L.shape
    (ph, pw), st = L.padding, L.stride
    y = e["o"]["y"].reshape(L.out_shape)
    if L.act == 3:
        _positive(pkg, y, e["name"])
    x = pkg.bf16_bits_to_f32(a["x"]).reshape(N, H, W, C)
    want = pkg.f32_to_bf16_bits(DR.fwd(x, pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(a["filt"])), a["bias"], st, ph, pw, L.act))
    return {"y": _exact(y, want, e["name"] + " y")}


def dwconv_backward(pkg, e, full):
    L, a, o = e["layer"], e["a"], e["o"]
    N, H, W, C, R, S = L.shape
    (ph, pw), st = L.padding, L.stride
    r = {"dpre": _dpre(pkg, e, L.act, e["name"])}
    d = pkg.bf16_bits_to_f32(o["dy"]).reshape(L.out_shape)
    if o.get("dx") is not None:
        wq = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(a["filt"]))
        r["dx"] = _exact(o["dx"].reshape(N, H, W, C), pkg.f32_to_bf16_bits(DR.dgrad(d, wq, H, W, st, ph, pw)[0]), e["name"] + " dx")
    if full:
        x = pkg.bf16_bits_to_f32(a["_x"]).reshape(N, H, W, C)
        r["dw"] = _ratio(o["dw"] - DR.wgrad_f64(x, d, R, S, st, ph, pw), 2 * L.info["n_acc"] * U * DR.wgrad_abs_f64(x, d, R, S, st, ph, pw))
    return r


def bn_forward(pkg, e, full):
    L, a, o = e["layer"], e["a"], e["o"]
    N, H, W, C = L.shape
    M = L.pixels
    xb = a["x"].reshape(M, C)
    rb = None if a.get("r") is None else a["r"].reshape(M, C)
    y = o["y"].reshape(M, C)
    if L.act == 3:
        _positive(pkg, y, e["name"])
    r = {}
    if e["argv"]["training"]:
        mean, rstd = o["save_mean"], o["save_rstd"]
        r["y"] = _exact(y, BR.fwd_bits(pkg, xb, a["gamma"], a["beta"], mean, rstd, rb, L.act), e["name"] + " y")
        r["running_mean"] = _exact(o["running_mean"], BR.running_update(a["running_mean"], mean, L.momentum), e["name"] + " running_mean")
        # the statistics on every pass (full or not): the running-variance chain over the steps reads e["stats"]
        m64, v64, vb = BR.check_stats(pkg, xb, mean, rstd, L.eps)
        e["stats"] = dict(v64=v64, var_bound=vb)
        x = pkg.bf16_bits_to_f32(xb).astype(np.float64)
        r["mean"] = _ratio(mean - m64, BR.n_stat(pkg, M, C) * U * (x.max(0) - x.min(0)) + U * np.abs(m64))
        r["var"] = _ratio(1.0 / rstd.astype(np.float64) ** 2 - np.float64(np.float32(L.eps)) - v64, vb)
    else:
        rm, rv = a["running_mean"], a["running_var"]
        r["eval y"] = _exact(y, BR.fwd_bits(pkg, xb, a["gamma"], a["beta"], rm, BR.eval_rstd(rv, L.eps), rb, L.act), e["name"] + " eval y")
        _exact(o["running_mean"].view(np.uint32), rm.view(np.uint32), e["name"] + " eval running_mean")
        _exact(o["running_var"].view(np.uint32), rv.view(np.uint32), e["name"] + " eval running_var")
    return r


def bn_backward(pkg, e, full):
    L, a, o, argv = e["layer"], e["a"], e["o"], e["argv"]
    N, H, W, C = L.shape
    M = L.pixels
    xb, yb, dyb = a["_x"].reshape(M, C), a["y"].reshape(M, C), a["dy"].reshape(M, C)
    dy2b = None if a.get("dy2") is None else a["dy2"].reshape(M, C)
    g = BR.grad_bits(pkg, yb, dyb, dy2b, L.act)
    r = {}
    if o.get("dr") is not None:
        r["dr"] = _exact(o["dr"].reshape(M, C), g, e["name"] + " dr")
    mean, rstd = a["save_mean"], a["save_rstd"]
    want = BR.dx_bits(pkg, xb, g, a["gamma"], mean, rstd, o["dgamma"], o["dbeta"])
    r["dx"] = _exact(o["dx"].reshape(M, C), want, e["name"] + " dx")
    if full:
        gf = pkg.bf16_bits_to_f32(g).astype(np.float64)
        xh = BR.xhat32(pkg, xb, mean, rstd).astype(np.float64)
        k = 2 * (BR.n_acc(pkg, M, C) + 1) * U
        r["dbeta"] = _ratio(o["dbeta"] - gf.sum(0), k * np.abs(gf).sum(0))
        r["dgamma"] = _ratio(o["dgamma"] - (gf * xh).sum(0), k * np.abs(gf * xh).sum(0))
    return r


def _pool_geometry(L):
    N, H, W, C, R, S = L.shape
    return N, H, W, C, R, S, L.stride, L.padding[0], L.padding[1], L.out_shape[1], L.out_shape[2]


def maxpool_forward(pkg, e, full):
    L = e["layer"]
    N, H, W, C, R, S, st, ph, pw, P, Q = _pool_geometry(L)
    xb = e["a"]["x"].reshape(N, H, W, C)
    am = MR.fwd_argmax(pkg.bf16_bits_to_f32(xb), R, S, st, ph, pw)
    r = {"argmax": _exact(e["o"]["argmax"], am, e["name"] + " argmax")}
    y = _img(e["o"]["y"], N, L.image_rows or P, L.row_pitch, P, Q * C).reshape(N, P, Q, C)
    r["y"] = _exact(y, MR.gather(xb, am, S, st, ph, pw), e["name"] + " y")
    return r


def maxpool_backward(pkg, e, full):
    L = e["layer"]
    N, H, W, C, R, S, st, ph, pw, P, Q = _pool_geometry(L)
    dy = _img(e["a"]["dy"], N, L.image_rows or P, L.row_pitch, P, Q * C).reshape(N, P, Q, C)
    want = MR.bwd_bf16(pkg, dy, e["a"]["argmax"].astype(np.int64), H, W, R, S, st, ph, pw)
    return {"dx": _exact(e["o"]["dx"].reshape(N, H, W, C), want, e["name"] + " dx")}


def avgpool_forward(pkg, e, full):
    L = e["layer"]
    N, H, W, C, R, S, st, ph, pw, P, Q = _pool_geometry(L)
    x = pkg.bf16_bits_to_f32(e["a"]["x"]).reshape(N, H, W, C)
    y = _img(e["o"]["y"], N, L.image_rows or P, L.row_pitch, P, Q * C).reshape(N, P, Q, C)
    return {"y": _exact(y, pkg.f32_to_bf16_bits(AR.fwd(x, R, S, st, ph, pw, L.count_include_pad)), e["name"] + " y")}


def avgpool_backward(pkg, e, full):
    L = e["layer"]
    N, H, W, C, R, S, st, ph, pw, P, Q = _pool_geometry(L)
    dy = pkg.bf16_bits_to_f32(_img(e["a"]["dy"], N, L.image_rows or P, L.row_pitch, P, Q * C)).reshape(N, P, Q, C)
    want = pkg.f32_to_bf16_bits(AR.bwd(dy, H, W, R, S, st, ph, pw, L.count_include_pad)[0])
    return {"dx": _exact(e["o"]["dx"].reshape(N, H, W, C), want, e["name"] + " dx")}


def gap_forward(pkg, e, full):
    L = e["layer"]
    N, H, W, C = L.shape
    if not full:
        return {}
    x = pkg.bf16_bits_to_f32(e["a"]["x"]).reshape(N, H, W, C)
    y = pkg.bf16_bits_to_f32(e["o"]["y"].reshape(N, L.row_pitch)[:, :C])
    m, E, lo, hi = AR.gap_bound(pkg, x, L.info)
    assert np.all((y >= lo) & (y <= hi)), e["name"] + " y outside its bound"
    # reported: |y - m| over E plus half a bf16 ulp (the rounding lo and hi carry)
    half_ulp = np.exp2(np.floor(np.log2(np.maximum(np.maximum(np.abs(y), np.abs(m)), 2.0 ** -126))) - 8)
    return {"y": _ratio(y - m, E + half_ulp)}


def gap_backward(pkg, e, full):
    L = e["layer"]
    N, H, W, C = L.shape
    dy = pkg.bf16_bits_to_f32(e["a"]["dy"].reshape(N, L.row_pitch)[:, :C])
    return {"dx": _exact(e["o"]["dx"].reshape(N, H, W, C), pkg.f32_to_bf16_bits(AR.global_bwd(dy, H, W)), e["name"] + " dx")}


def softmax(pkg, e, full):
    """dz bit-identical to float64 -> fp32 -> bf16, one ulp allowed only within 1e-12 of a rounding boundary (counted as
    "one-ulp"); loss within 1e-6 and pred exact"""
    argv, a, o = e["argv"], e["a"], e["o"]
    N, O = argv["N"], argv["O"]
    z = pkg.bf16_bits_to_f32(a["logits"].reshape(N, O))
    g, lref, pref = LR.softmax_ce_f64(z, a["labels"], np.float32(argv["scale"]))
    want = LR.f64_to_bf16_bits(pkg, g)
    diff = np.abs(o["dlogits"].reshape(N, O).astype(np.int64) - want.astype(np.int64))
    near = LR.near_boundary(pkg, g)
    assert np.all((diff == 0) | (near & (diff <= 1))), "dz differs away from a rounding boundary"
    r = {"dz": 0.0, "one-ulp": int((diff != 0).sum())}
    if o.get("loss") is not None:
        r["loss"] = _ratio(o["loss"] - lref, 1e-6 * np.maximum(1.0, np.abs(lref)))
    if o.get("pred") is not None:
        r["pred"] = _exact(o["pred"], pref, "pred")
    return r


CHECKERS = {("ConvLayer", "forward"): conv_forward, ("ConvLayer", "backward"): conv_backward,
            ("LinearLayer", "forward"): linear_forward, ("LinearLayer", "backward"): linear_backward,
            ("DepthwiseConvLayer", "forward"): dwconv_forward, ("DepthwiseConvLayer", "backward"): dwconv_backward,
            ("BatchNormLayer", "forward"): bn_forward, ("BatchNormLayer", "backward"): bn_backward,
            ("MaxPoolLayer", "forward"): maxpool_forward, ("MaxPoolLayer", "backward"): maxpool_backward,
            ("AvgPoolLayer", "forward"): avgpool_forward, ("AvgPoolLayer", "backward"): avgpool_backward,
            ("GlobalAvgPoolLayer", "forward"): gap_forward, ("GlobalAvgPoolLayer", "backward"): gap_backward,
            ("softmax", "softmax"): softmax}


def check(pkg, e, full=True):
    """run the entry's checker; returns {check name: worst ratio to its bound} (the one-ulp softmax count as an int)"""
    return CHECKERS[(e["kind"], e["op"])](pkg, e, full)
