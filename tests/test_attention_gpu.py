"""Self-attention on the device (pcnn_attention_bf16_fwd / _bwd): o, lse, dq, dk and dv against the float64 reference of
attention_ref.py within its stated error bounds, for every head size, 1, 2 and 4 heads, T from 1 to 3136 (ragged last blocks of
1, 36, 49, 16, 4, 16 and 0 keys), the fused qkv layout and the four shapes scripts/conv_bench.py attn times (there a seeded subset
of images is checked: each image is computed on its own).  Reruns are bit-identical; an image alone equals the same image in a
batch, and one head's bits do not depend on the other heads; NaN canaries past the outputs and in unwritten columns of a shared
dq/dk/dv buffer survive; a SelfAttentionLayer step checks both projections' dw, db and dx against float64 on the layer's own
operands under SGD and AdamW."""
import math

import numpy as np
import pytest

import attention_ref as A
from example_nets import NAN_BF16

pytestmark = pytest.mark.gpu

TAIL = 64


def to_bits(pkg, a):
    return pkg.f32_to_bf16_bits(np.asarray(a, np.float32))


class Case:
    """q, k, v in one fused [N][T][ld] buffer (columns 0, h d, 2 h d) or three dense ones; dout dense.  Outputs NaN-prefilled."""

    def __init__(self, eng, pkg, rng, N, T, h, d, fused=False, pad=0, scale=None):
        self.eng, self.pkg = eng, pkg
        self.N, self.T, self.h, self.d = N, T, h, d
        self.scale = 1.0 / math.sqrt(d) if scale is None else scale
        hd = h * d
        g = lambda: A.bf16(rng.standard_normal((N, T, h, d)).astype(np.float32))
        self.q, self.k, self.v, self.dout = g(), g(), g(), g()
        self.fused = fused
        if fused:
            self.ld = 3 * hd + pad
            buf = np.full((N * T, self.ld), NAN_BF16, np.uint16)
            for i, a in enumerate((self.q, self.k, self.v)):
                buf[:, i * hd:(i + 1) * hd] = to_bits(pkg, a.reshape(N * T, hd))
            self.qkv = eng.to_device(np.concatenate([buf.ravel(), np.full(TAIL, NAN_BF16, np.uint16)]))
            base = self.qkv.ptr
            self.qp, self.kp, self.vp = base, base + 2 * hd, base + 4 * hd
        else:
            self.ld = hd
            self.bufs = [eng.to_device(np.concatenate([to_bits(pkg, a).ravel(), np.full(TAIL, NAN_BF16, np.uint16)]))
                         for a in (self.q, self.k, self.v)]
            self.qp, self.kp, self.vp = (b.ptr for b in self.bufs)
        self.dod = eng.to_device(to_bits(pkg, self.dout).ravel())

    def run(self):
        """o [N][T][h][d] (float32 of the bf16), lse, dq, dk, dv; plus the raw buffers with their tails"""
        N, T, h, d, hd = self.N, self.T, self.h, self.d, self.h * self.d
        od = self.eng.to_device(np.full(N * T * hd + TAIL, NAN_BF16, np.uint16))
        lsed = self.eng.to_device(np.full(N * h * T + TAIL, np.nan, np.float32))
        self.eng.attention_fwd(self.qp, self.kp, self.vp, od, lsed, N, T, h, d, ld=self.ld, scale=self.scale)
        ldg = self.ld if self.fused else hd          # a padded fused layout leaves columns 3 h d .. ld_g of dq/dk/dv unwritten
        if self.fused:
            g = self.eng.to_device(np.full(N * T * ldg + TAIL, NAN_BF16, np.uint16))
            gp = (g.ptr, g.ptr + 2 * hd, g.ptr + 4 * hd)
            gb = [g]
        else:
            gb = [self.eng.to_device(np.full(N * T * hd + TAIL, NAN_BF16, np.uint16)) for _ in range(3)]
            gp = tuple(b.ptr for b in gb)
        self.eng.attention_bwd(self.qp, self.kp, self.vp, od, self.dod, lsed, *gp, N, T, h, d, ld=self.ld, ld_g=ldg, scale=self.scale)
        self.eng.sync()
        o_raw, lse_raw = od.to_host(), lsed.to_host()
        g_raw = [b.to_host() for b in gb]
        f = self.pkg.bf16_bits_to_f32
        o = f(o_raw[:N * T * hd]).reshape(N, T, h, d)
        lse = lse_raw[:N * h * T].reshape(N, h, T)
        if self.fused:
            full = f(g_raw[0][:N * T * ldg]).reshape(N * T, ldg)
            grads = [full[:, i * hd:(i + 1) * hd].reshape(N, T, h, d) for i in range(3)]
        else:
            grads = [f(r[:N * T * hd]).reshape(N, T, h, d) for r in g_raw]
        return dict(o=o, lse=lse, dq=grads[0], dk=grads[1], dv=grads[2]), (o_raw, lse_raw, g_raw)

    def check(self, out, images=None, limit=1.0):
        sel = np.arange(self.N) if images is None else np.asarray(images)
        b = A.bounds(self.q[sel], self.k[sel], self.v[sel], self.dout[sel], self.scale)
        worst = {}
        for name, (ref, bound) in b.items():
            worst[name] = A.worst(out[name][sel], ref, bound)
        assert max(worst.values()) <= limit, (self.N, self.T, self.h, self.d, worst)
        return worst


SHAPES = [(2, T, h, d) for d in (16, 32, 64, 128) for T, h in ((1, 1), (36, 2), (49, 4), (144, 1), (196, 2))] + \
         [(2, 784, 1, 16), (2, 784, 2, 64), (1, 784, 1, 128), (1, 3136, 1, 64), (1, 3136, 2, 16)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "N%d-T%d-h%d-d%d" % s)
def test_against_float64(eng, pkg, shape):
    rng = np.random.default_rng(sum(shape))
    c = Case(eng, pkg, rng, *shape)
    out, _ = c.run()
    c.check(out)


@pytest.mark.parametrize("h,d,pad", [(1, 16, 0), (2, 32, 0), (4, 16, 8), (5, 16, 0), (1, 64, 16)])
def test_fused_layout(eng, pkg, h, d, pad):
    """q, k and v as the column blocks of one projection output (ld = 3 h d, or wider), and dq, dk, dv into one shared buffer"""
    rng = np.random.default_rng(h * d + pad)
    c = Case(eng, pkg, rng, 3, 144, h, d, fused=True, pad=pad)
    out, _ = c.run()
    c.check(out)


@pytest.mark.parametrize("N,T,h,d", [(128, 196, 4, 64), (32, 784, 1, 128), (16, 3136, 1, 64), (8, 4096, 1, 64)])
def test_benchmark_shapes(eng, pkg, N, T, h, d):
    """the shapes conv_bench.py attn times, many tiles per CTA on 132 SMs; two seeded images checked"""
    rng = np.random.default_rng(N + T)
    c = Case(eng, pkg, rng, N, T, h, d)
    info = pkg.attention_info(N, T, h, d)
    assert info["fwd_tiles"] > 132
    out, _ = c.run()
    c.check(out, images=np.sort(rng.choice(N, 2, replace=False)))


def test_large_logits_and_dominant_key(eng, pkg):
    """logits near +-10^4 (the max subtraction decides everything) and one key that takes all the weight"""
    rng = np.random.default_rng(7)
    c = Case(eng, pkg, rng, 2, 144, 1, 16, scale=1.0)
    q = np.zeros_like(c.q)
    k = np.zeros_like(c.k)
    q[..., 0] = 100.0
    k[..., 0] = A.bf16(np.round(rng.uniform(-100, 98.4, k.shape[:-1])).astype(np.float32))
    k[:, 77, :, 0] = 100.0                               # the dominant key: logit 10^4
    c.q, c.k = q, k
    c.bufs[0].copy_from(np.concatenate([to_bits(pkg, q).ravel(), np.full(TAIL, NAN_BF16, np.uint16)]))
    c.bufs[1].copy_from(np.concatenate([to_bits(pkg, k).ravel(), np.full(TAIL, NAN_BF16, np.uint16)]))
    out, _ = c.run()
    c.check(out)
    assert np.all(out["o"][:, :, 0] == c.v[:, 77:78, 0])


def test_rerun_bit_identical(eng, pkg):
    rng = np.random.default_rng(3)
    c = Case(eng, pkg, rng, 4, 196, 2, 32)
    _, a = c.run()
    _, b = c.run()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1], equal_nan=True)
    assert all(np.array_equal(x, y) for x, y in zip(a[2], b[2]))


def test_image_alone_and_heads_independent(eng, pkg):
    """image 5 of a batch of 9 equals the same image run alone; head 1 of 4 equals that head run with h = 1"""
    rng = np.random.default_rng(11)
    big = Case(eng, pkg, rng, 9, 144, 4, 16)
    out, _ = big.run()
    one = Case(eng, pkg, rng, 1, 144, 4, 16)
    one.q, one.k, one.v, one.dout = (a[5:6] for a in (big.q, big.k, big.v, big.dout))
    for buf, a in zip(one.bufs, (one.q, one.k, one.v)):
        buf.copy_from(np.concatenate([to_bits(pkg, a).ravel(), np.full(TAIL, NAN_BF16, np.uint16)]))
    one.dod.copy_from(to_bits(pkg, one.dout).ravel())
    alone, _ = one.run()
    for name in ("o", "lse", "dq", "dk", "dv"):
        assert np.array_equal(alone[name][0], out[name][5]), name
    head = Case(eng, pkg, rng, 9, 144, 1, 16)
    head.q, head.k, head.v, head.dout = (np.ascontiguousarray(a[:, :, 1:2]) for a in (big.q, big.k, big.v, big.dout))
    for buf, a in zip(head.bufs, (head.q, head.k, head.v)):
        buf.copy_from(np.concatenate([to_bits(pkg, a).ravel(), np.full(TAIL, NAN_BF16, np.uint16)]))
    head.dod.copy_from(to_bits(pkg, head.dout).ravel())
    h1, _ = head.run()
    for name in ("o", "dq", "dk", "dv"):
        assert np.array_equal(h1[name][:, :, 0], out[name][:, :, 1]), name
    assert np.array_equal(h1["lse"][:, 0], out["lse"][:, 1])


def test_canaries(eng, pkg):
    """nothing past N T rows of o and lse is written, nor the 8 padding columns of every row of a shared dq/dk/dv buffer with
    ld_g = 3 h d + 8, nor anything past its last row"""
    rng = np.random.default_rng(5)
    c = Case(eng, pkg, rng, 2, 49, 2, 16, fused=True, pad=8)
    hd = 32
    N, T = 2, 49
    c.run()
    out, (o_raw, lse_raw, g_raw) = c.run()
    assert np.all(o_raw[N * T * hd:] == NAN_BF16) and np.all(np.isnan(lse_raw[N * 2 * T:]))
    g = g_raw[0]
    ldg = 3 * hd + 8
    assert np.all(g[N * T * ldg:] == NAN_BF16)
    assert np.all(g[:N * T * ldg].reshape(N * T, ldg)[:, 3 * hd:] == NAN_BF16)
    assert not np.any(np.isnan(out["dq"])) and not np.any(np.isnan(out["dv"]))


def test_refusals(eng, pkg):
    a = eng.array(4096, np.uint16)
    lse = eng.array(1024)
    with pytest.raises(pkg.PcnnError, match="pcnn_attention_bf16_fwd: head size d = 48"):
        eng.attention_fwd(a, a, a, a, lse, 1, 4, 1, 48)
    with pytest.raises(pkg.PcnnError, match="pcnn_attention_bf16_fwd: o or lse overlaps"):
        eng.attention_fwd(a, a, a, a, lse, 1, 4, 1, 16)
    with pytest.raises(pkg.PcnnError, match="pcnn_attention_bf16_bwd: dq, dk and dv may share a buffer only on disjoint columns"):
        g = eng.array(4096, np.uint16)
        eng.attention_bwd(a, a, a, a, a, lse, g, g.ptr + 16, g.ptr + 64, 1, 4, 1, 16, ld_g=48)


def _layer_operands(layer):
    f = lambda a: a.to_host().astype(np.uint16)
    return f(layer.qkv_y), f(layer.o), f(layer.do), f(layer.dqkv)


@pytest.mark.parametrize("opt", ["sgd", "adamw"])
def test_layer_step(eng, pkg, opt):
    """one SelfAttentionLayer step: the core on the layer's own operands within the bounds, both projections' dw, db and dx
    against float64 on the same operands, and one optimizer step"""
    N, H, W, C, h, d = 4, 12, 12, 16, 1, 16
    hd, T = h * d, H * W
    rng = np.random.default_rng(1 if opt == "sgd" else 2)
    wq = (rng.standard_normal((3 * hd, C)) / math.sqrt(C)).astype(np.float32)
    bq = (rng.standard_normal(3 * hd) * 0.1).astype(np.float32)
    wo = (rng.standard_normal((C, hd)) / math.sqrt(hd)).astype(np.float32)
    bo = (rng.standard_normal(C) * 0.1).astype(np.float32)
    layer = pkg.SelfAttentionLayer(eng, N, H, W, C, h, d, wq, bq, wo, bo)
    x = to_bits(pkg, rng.standard_normal((N, H, W, C)))
    dy = to_bits(pkg, rng.standard_normal((N, H, W, C)))
    xd, dyd = eng.to_device(x.ravel()), eng.to_device(dy.ravel())
    yd, dxd = eng.array(x.size, np.uint16), eng.array(x.size, np.uint16)
    layer.forward(xd, yd)
    layer.backward(dyd, dxd)
    eng.sync()
    f = pkg.bf16_bits_to_f32
    qkv, o, do, dqkv = (f(a).astype(np.float64) for a in _layer_operands(layer))
    qkv = qkv.reshape(N, T, 3, h, d)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    b = A.bounds(q, k, v, do.reshape(N, T, h, d), 1 / math.sqrt(d))
    got = dict(o=o.reshape(N, T, h, d), dq=dqkv.reshape(N, T, 3, h, d)[:, :, 0], dk=dqkv.reshape(N, T, 3, h, d)[:, :, 1],
               dv=dqkv.reshape(N, T, 3, h, d)[:, :, 2], lse=layer.lse.to_host().reshape(N, h, T))
    for name, (ref, bound) in b.items():
        assert A.worst(got[name], ref, bound) <= 1.0, name
    xf, dyf = f(x).astype(np.float64).reshape(N * T, C), f(dy).astype(np.float64).reshape(N * T, C)
    rows = N * T
    wqb, wob = A.bf16(wq).astype(np.float64), A.bf16(wo).astype(np.float64)
    o2, do2, dqkv2 = o.reshape(rows, hd), do.reshape(rows, hd), dqkv.reshape(rows, 3 * hd)
    # fp32 sums over at most `rows` terms, bf16 outputs
    tol = lambda terms, ref: rows * 2.0 ** -23 * terms + 2.0 ** -8 * np.abs(ref)
    checks = [
        (layer.out.dw.to_host().reshape(C, hd), dyf.T @ o2, np.abs(dyf).T @ np.abs(o2)),
        (layer.out.db.to_host(), dyf.sum(0), np.abs(dyf).sum(0)),
        (f(layer.do.to_host()).reshape(rows, hd), dyf @ wob, np.abs(dyf) @ np.abs(wob)),
        (layer.qkv.dw.to_host().reshape(3 * hd, C), dqkv2.T @ xf, np.abs(dqkv2).T @ np.abs(xf)),
        (layer.qkv.db.to_host(), dqkv2.sum(0), np.abs(dqkv2).sum(0)),
        (f(dxd.to_host()).reshape(rows, C), dqkv2 @ wqb, np.abs(dqkv2) @ np.abs(wqb)),
    ]
    for i, (got_, ref, terms) in enumerate(checks):
        assert np.all(np.abs(got_ - ref) <= tol(terms, ref) + 1e-30), i
    assert np.array_equal(dyd.to_host(), dy.ravel())                 # dy left unchanged
    before = [t[0].to_host().copy() for t in layer.optim_tensors()]
    grads = [t[1].to_host().copy() for t in layer.optim_tensors()]
    lr = 0.05
    optim = pkg.SGD(eng, [layer]) if opt == "sgd" else pkg.AdamW(eng, [layer], weight_decay=0.0)
    optim.step(lr)
    eng.sync()
    after = [t[0].to_host() for t in layer.optim_tensors()]
    for w0, g, w1 in zip(before, grads, after):
        if opt == "sgd":
            want = w0.astype(np.float64) - lr * g
        else:   # Adam's first step moves every weight with a nonzero gradient by lr sign(g) (eps aside)
            want = w0.astype(np.float64) - lr * g / (np.abs(g) + 1e-8)
        assert np.allclose(w1, want, rtol=1e-5, atol=1e-6)
    layer.close()
