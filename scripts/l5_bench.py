#!/usr/bin/env python
"""scripts/l5_bench.py -- training-step time of the LeNet-5-style variant (csrc/lenet5_kernels.cu: c1 -> s2 -> c3 16@5x5x6
-> s4 -> f 256->10, 5152 parameters; SURVEY.md 8f row 4) at 1, 64, 256 and 1024 images per step.  One step =
pcnn_l5_train_step (fused forward+backward kernel + reduce/update kernel), device-resident u8 pixels walked through a set
larger than the L2, CUDA events on the launching stream after warm-up.  Useful flops per image (forward + both backward
products, multiply-add = 2): c1 2*6*576*25*3 (no input gradient: 2 products), c3 2*16*64*150*3, f 2*10*256*3."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pcnn_loader  # noqa: E402

pkg = pcnn_loader.load()
torch.cuda.set_device(0)
stream = torch.cuda.Stream()
torch.cuda.set_stream(stream)
eng = pkg.Engine(0, stream.cuda_stream)
rng = np.random.default_rng(7)
NPARAM = 5152
FLOPS_PER_IMAGE = 2 * 6 * 576 * 25 * 2 + 2 * 16 * 64 * 150 * 3 + 2 * 10 * 256 * 3 + 2 * 6 * 144 * 16 * 3
NSET = 262144                                               # 205 MB of u8 pixels > 50 MB L2

imgs = torch.randint(0, 256, (NSET, 784), dtype=torch.uint8, device="cuda")
labs = torch.randint(0, 10, (NSET,), dtype=torch.uint8, device="cuda")
p0 = rng.uniform(-0.5, 0.5, NPARAM).astype(np.float32)
for B in (1, 64, 256, 1024):
    params = eng.to_device(p0)
    iters = 400 if B <= 256 else 200
    span = NSET // B

    def step(i):
        lo = (i % span) * B
        eng.l5_train_step(params, imgs[lo:lo + B], pkg.U8, labs[lo:lo + B], B)

    for i in range(10):
        step(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for i in range(iters):
        step(10 + i)
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    print(json.dumps({"case": "lenet5_variant_train_step", "batch": B, "us_per_step": ms * 1e3, "img_per_s": B / (ms * 1e-3),
                      "useful_TFLOPs": FLOPS_PER_IMAGE * B / (ms * 1e-3) / 1e12, "launches_per_step": 2,
                      "note": "stream-ordered launches from Python; small batches are launch-bound"}), flush=True)
