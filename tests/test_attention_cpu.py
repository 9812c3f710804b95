"""Self-attention without a GPU: the float64 reference of attention_ref.py against torch's float64 scaled_dot_product_attention and
autograd (ragged T, several heads, a strided fused-qkv layout, T = 1); pcnn_attention_info's partition and its refusals, one
message per domain rule, each naming the called function; and the float32 / bf16 emulation of the operation order include/pcnn.h
states inside the error bounds the GPU tests use, on random inputs, logits of +-10^4 and one dominant key."""
import math
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import attention_ref as A


def _torch(q, k, v, dout, scale):
    t = [torch.tensor(np.transpose(a, (0, 2, 1, 3)), dtype=torch.float64, requires_grad=True) for a in (q, k, v)]
    o = F.scaled_dot_product_attention(*t, scale=scale)
    o.backward(torch.tensor(np.transpose(dout, (0, 2, 1, 3)), dtype=torch.float64))
    back = lambda x: np.transpose(x.detach().numpy(), (0, 2, 1, 3))
    lse = torch.logsumexp(t[0] @ t[1].transpose(-1, -2) * scale, -1)
    return back(o), lse.detach().numpy(), back(t[0].grad), back(t[1].grad), back(t[2].grad)


@pytest.mark.parametrize("N,T,h,d", [(2, 1, 1, 16), (2, 37, 2, 16), (1, 144, 1, 32), (3, 49, 4, 16), (1, 130, 2, 64)])
def test_reference_matches_torch(N, T, h, d):
    rng = np.random.default_rng(N * T + h * d)
    q, k, v, dout = (rng.standard_normal((N, T, h, d)) for _ in range(4))
    scale = 1 / math.sqrt(d)
    o, lse, _ = A.forward(q, k, v, scale)
    dq, dk, dv = A.backward(q, k, v, dout, scale)[:3]
    want = _torch(q, k, v, dout, scale)
    for got, ref in zip((o, lse, dq, dk, dv), want):
        assert np.allclose(got, ref, rtol=1e-12, atol=1e-12)


def test_reference_fused_layout():
    """q, k, v taken as strided column blocks of one [N T][3 h d + 8] projection equal the dense ones"""
    rng = np.random.default_rng(4)
    N, T, h, d = 2, 36, 2, 16
    buf = rng.standard_normal((N * T, 3 * h * d + 8))
    q, k, v = (buf[:, i * h * d:(i + 1) * h * d].reshape(N, T, h, d) for i in range(3))
    dout = rng.standard_normal((N, T, h, d))
    got = A.backward(q, k, v, dout, 0.3)[:3]
    want = _torch(np.ascontiguousarray(q), np.ascontiguousarray(k), np.ascontiguousarray(v), dout, 0.3)[2:]
    for g, w in zip(got, want):
        assert np.allclose(g, w, rtol=1e-12, atol=1e-12)


def test_info_partition(pkg):
    i = pkg.attention_info(128, 196, 4, 64)
    assert (i["query_rows"], i["block_rows"], i["stages"]) == (128, 64, 2)
    assert i["fwd_tiles"] == i["dq_tiles"] == i["dkdv_tiles"] == 128 * 4 * 2
    assert i["scratch_bytes"] == 128 * 4 * 196 * 4
    assert pkg.attention_info(1, 1, 1, 16)["fwd_tiles"] == 1
    # the partition of one (image, head) does not change with N or the other heads
    assert pkg.attention_info(7, 144, 3, 16)["fwd_tiles"] == 7 * 3 * pkg.attention_info(1, 144, 1, 16)["fwd_tiles"]


@pytest.mark.parametrize("args,rule", [
    (dict(d=48), "head size d = 48: 16, 32, 64 or 128"),
    (dict(heads=0), "heads = 0: at least 1"),
    (dict(N=0), "N = 0: at least one image"),
    (dict(T=0), "T = 0 tokens: 1 <= T <= 16384"),
    (dict(T=16385), "T = 16385 tokens"),
    (dict(ld=60), "ld = 60: a multiple of 8"),
    (dict(ld=68), "ld = 68: a multiple of 8"),
    (dict(ld_g=8), "ld_g = 8: a multiple of 8"),
    (dict(ld_g=100), "ld_g = 100"),
    (dict(scale=0.0), "scale = 0: a finite scale > 0"),
    (dict(scale=float("inf")), "scale = inf"),
    (dict(N=1 << 30, heads=4, T=16384, ld=256), "N * heads * ceil(T / 128) = 549755813888 tiles: fewer than 2^31"),
])
def test_info_refusals(pkg, args, rule):
    a = dict(N=2, T=144, heads=1, d=64, ld=64, ld_g=0, scale=0.125)
    a.update(args)
    with pytest.raises(pkg.PcnnError, match=re.escape("pcnn_attention_info: " + rule)):
        pkg.attention_info(a["N"], a["T"], a["heads"], a["d"], a["ld"], a["ld_g"], a["scale"])


def test_device_calls_refuse_null_arguments(pkg):
    """the two device calls check their arguments before any GPU work (their shape rules are info's: one function makes both)"""
    L = pkg.lib()
    assert L.pcnn_attention_bf16_fwd(None, None, None, None, 1, 1, 1, 16, 16, 1.0, None, None) != 0
    assert L.pcnn_last_error_string().decode().startswith("pcnn_attention_bf16_fwd: NULL argument")
    assert L.pcnn_attention_bf16_bwd(None, None, None, None, None, None, None, 1, 1, 1, 16, 16, 1.0, None, None, None, 16) != 0
    assert L.pcnn_last_error_string().decode().startswith("pcnn_attention_bf16_bwd: NULL argument")


def _bf16_inputs(rng, N, T, h, d, mult=1.0):
    return [A.bf16((rng.standard_normal((N, T, h, d)) * mult).astype(np.float32)) for _ in range(4)]


def _inside(q, k, v, dout, scale):
    b = A.bounds(q, k, v, dout, scale)
    got = dict(zip(("o", "lse", "dq", "dk", "dv"), A.emulate(q, k, v, dout, scale)))
    w = {n: A.worst(got[n], *b[n]) for n in b}
    assert max(w.values()) <= 1.0, w
    return w


@pytest.mark.parametrize("N,T,h,d", [(2, 1, 1, 16), (2, 36, 2, 32), (1, 144, 1, 16), (1, 196, 2, 64), (1, 200, 1, 128)])
def test_emulation_inside_bounds_random(N, T, h, d):
    rng = np.random.default_rng(T + d)
    _inside(*_bf16_inputs(rng, N, T, h, d), 1 / math.sqrt(d))


def test_emulation_inside_bounds_large_logits():
    """scores of +-10^4 from exact products: without the max subtraction every exponent would overflow"""
    rng = np.random.default_rng(9)
    N, T, h, d = 2, 144, 1, 16
    q, k, v, dout = _bf16_inputs(rng, N, T, h, d)
    q[:] = 0
    k[:] = 0
    q[..., 0] = 100.0
    k[..., 0] = np.round(rng.uniform(-100, 98.4, (N, T, h)))
    k[:, 77, :, 0] = 100.0                                # one key 100 above the rest in every row: the GPU test's input
    _inside(q, k, v, dout, 1.0)


def test_emulation_inside_bounds_tied_large_logits():
    """scores of +-10^4 with several keys tied at the maximum: dS k cancels over the tied keys, and the bf16 O in D does not"""
    rng = np.random.default_rng(9)
    N, T, h, d = 2, 144, 1, 16
    q, k, v, dout = _bf16_inputs(rng, N, T, h, d)
    q[:] = 0
    k[:] = 0
    q[..., 0] = 100.0
    k[..., 0] = np.round(rng.uniform(-100, 98.4, (N, T, h)))
    k[:, 10:13, :, 0] = 99.0                              # three keys tied at the maximum logit 9900
    _inside(q, k, v, dout, 1.0)


def test_emulation_inside_bounds_dominant_key():
    rng = np.random.default_rng(10)
    N, T, h, d = 1, 130, 2, 32
    q, k, v, dout = _bf16_inputs(rng, N, T, h, d)
    k[:, 77] = A.bf16(q.mean(1) * 8)                       # one key aligned with every query
    _inside(q, k, v, dout, 1 / math.sqrt(d))
