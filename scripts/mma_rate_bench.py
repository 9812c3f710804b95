#!/usr/bin/env python
"""scripts/mma_rate_bench.py -- SM clocks per wgmma product for the instruction shapes the convolution kernels can choose from."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pcnn_loader  # noqa: E402

pkg = pcnn_loader.load()
eng = pkg.Engine(0)
for (M, N) in ((64, 32), (128, 32), (128, 48), (128, 64), (128, 128), (128, 256), (64, 64), (64, 128), (64, 256)):
    for (a_mn, b_mn) in ((0, 0), (1, 0), (0, 1)):
        for nacc in (1, 2):
            if N * nacc > 512:
                continue
            clk = eng.measure_mma_rate(M, N, a_mn, b_mn, nacc, 2000)
            print(json.dumps({"M": M, "N": N, "K": 16, "a_major": "MN" if a_mn else "K", "b_major": "MN" if b_mn else "K", "accumulators": nacc,
                              "clk_per_mma": round(clk, 1), "mac_per_clk": round(M * N * 16 / clk, 1)}), flush=True)
eng.close()
