#!/usr/bin/env python
"""scripts/debug_conv_bwd.py -- one backward pass of the bf16 convolution (tensor-core path unless PCNN_CONV_BWD=fma) against the
oracle, with error statistics instead of an assert.  usage: debug_conv_bwd.py wgrad|dgrad N H W C K R S"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pcnn_loader  # noqa: E402
import oracle_lib as O  # noqa: E402

pkg = pcnn_loader.load()
what = sys.argv[1]
N, H, W, C, K, R, S = (int(v) for v in sys.argv[2:9])
P, Q = H - R + 1, W - S + 1
rng = np.random.default_rng(7)
x = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(0, 1, (N, H, W, C)).astype(np.float32)))
dy = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-1, 1, (N, P, Q, K)).astype(np.float32)))
f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
eng = pkg.Engine(0)
tag = {k: v for k, v in os.environ.items() if k.startswith("PCNN_")}
if what == "wgrad":
    ref = np.empty((K, R, S, C), np.float32)
    O.oracle().orc_conv_wgrad_nhwc(O.fp(x.reshape(-1)), O.fp(dy.reshape(-1)), O.fp(ref.reshape(-1)), N, H, W, C, K, R, S)
    dw = eng.array((K, R, S, C))
    eng.conv_wgrad(eng.to_device(pkg.f32_to_bf16_bits(x)), eng.to_device(pkg.f32_to_bf16_bits(dy)), dw, N, H, W, C, K, R, S)
    got = dw.to_host()
    rel = np.linalg.norm((got - ref).astype(np.float64)) / np.linalg.norm(ref.astype(np.float64))
    print("wgrad", sys.argv[2:9], tag, "rel-L2", rel, "ref[0,0,0,:]", ref[0, 0, 0], "got", got[0, 0, 0], flush=True)
    if rel > 1e-3:
        # which k rows match?  (diagnoses the row map of an M = 64 accumulator)
        for k in range(0, K, 8):
            e = np.abs(got[k] - ref[k]).max() / (np.abs(ref[k]).max() + 1e-9)
            print("  k", k, "max rel err", e)
else:
    ref = np.empty((N, H, W, C), np.float32)
    O.oracle().orc_conv_dgrad_nhwc(O.fp(dy.reshape(-1)), O.fp(f.reshape(-1)), O.fp(ref.reshape(-1)), N, H, W, C, K, R, S)
    dxo = eng.array((N, H, W, C), np.uint16)
    eng.conv_dgrad(eng.to_device(pkg.f32_to_bf16_bits(dy)), eng.to_device(f), dxo, N, H, W, C, K, R, S)
    got = pkg.bf16_bits_to_f32(dxo.to_host())
    bad = np.abs(got - ref) > 2.0 ** -8 * np.abs(ref) + 1e-3
    print("dgrad", sys.argv[2:9], tag, "bad", int(bad.sum()), "of", bad.size, "max abs err", float(np.abs(got - ref).max()), flush=True)
    if bad.any():
        idx = np.argwhere(bad)
        print("  first bad (n,h,w,c):", idx[:6].tolist())
        print("  bad rows h:", sorted(set(idx[:, 1].tolist()))[:40])
        print("  bad cols w:", sorted(set(idx[:, 2].tolist()))[:40])
        n, h, w, c = idx[0]
        print("  got", got[n, h, w], "ref", ref[n, h, w])
eng.close()
