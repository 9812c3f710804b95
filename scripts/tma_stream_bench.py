#!/usr/bin/env python
"""scripts/tma_stream_bench.py -- streaming-read ceiling of a TMA pipeline over dy [N,222,222,64] bf16 (config 5's big tensor) for the
box shapes of the convolution backward kernels (pcnn_measure_tma_read), next to the H100 SXM data-sheet HBM bandwidth (3.35 TB/s)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pcnn_loader  # noqa: E402

pkg = pcnn_loader.load()
torch.cuda.set_device(0)
eng = pkg.Engine(0)
N, P, Q = 128, 222, 222
buf = torch.zeros((N, P, Q, 64), dtype=torch.int16, device="cuda")
names = {0: "1-D bulk 16 KB", 1: "2-D box 64ch x 128px (16 KB contiguous)", 2: "dgrad pattern: 4 boxes 64ch x 1px x 32 rows",
         3: "wgrad pattern: box 64ch x 224px x 1 row (28 KB)"}
for mode in (0, 1, 2, 3):
    for stages in (os.environ.get("STAGES", "0").split(",")):
        if int(stages) > 0:
            os.environ["PCNN_DIAG_STAGES"] = stages
        gbps = eng.measure_tma_read(buf, N, P, Q, mode, 10)
        print(json.dumps({"mode": mode, "pattern": names[mode], "stages": stages, "GBps": gbps, "tensor_MB": buf.numel() * 2 / 1e6}), flush=True)
eng.close()
