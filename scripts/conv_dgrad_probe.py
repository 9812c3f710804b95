#!/usr/bin/env python
"""scripts/conv_dgrad_probe.py -- whether bench.py's conv block and scripts/conv_bench.py time the input gradient alike:
the same shape (config 5, N = 128) with the operands of either harness, in either order, plus fresh allocations."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pcnn_loader  # noqa: E402

pkg = pcnn_loader.load()
torch.cuda.set_device(0)
stream = torch.cuda.Stream()
torch.cuda.set_stream(stream)
eng = pkg.Engine(0, stream.cuda_stream)
N, H, W, C, K, R, S = 128, 224, 224, 3, 64, 3, 3
P, Q = H - R + 1, W - S + 1
alg = N * (H * W * C + P * Q * K) * 2


def timed(fn, iters=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(iters):
        fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


g = torch.Generator(device="cuda").manual_seed(1234)
x = torch.rand((N, H, W, C), device="cuda", generator=g).to(torch.bfloat16)
f = torch.rand((K, R, S, C), device="cuda", generator=g) - 0.5
y = torch.empty((N, P, Q, K), dtype=torch.bfloat16, device="cuda")
dx = torch.empty((N, H, W, C), dtype=torch.bfloat16, device="cuda")
plan = pkg.ConvPlan(eng, N, H, W, C, K, R, S, f.cpu().numpy(), None, act=0, row_pitch=W * C)
plan.fwd(x, y)
torch.cuda.synchronize()
rnd = torch.randint(0, 0x3F80, (N, P, Q, K), dtype=torch.int16, device="cuda")
rnd ^= (torch.randint(0, 2, (N, P, Q, K), dtype=torch.int16, device="cuda") << 15)
gauss = (torch.randn((N, P, Q, K), device="cuda", generator=g) * 0.5).to(torch.bfloat16)
zeros = torch.zeros((N, P, Q, K), dtype=torch.bfloat16, device="cuda")
for name, dy in (("forward output (bench.py)", y), ("random bit patterns (conv_bench.py)", rnd), ("gaussian 0.5", gauss), ("zeros", zeros),
                 ("forward output again", y)):
    ms = timed(lambda: eng.conv_dgrad(dy, f, dx, N, H, W, C, K, R, S))
    print(json.dumps({"dy": name, "ms": ms, "GBps": alg / (ms * 1e-3) / 1e9,
                      "absmax": float(dy.view(torch.bfloat16).float().abs().max()) if dy.dtype != torch.int16 else None}), flush=True)
plan.close()
eng.close()
