#!/usr/bin/env python
"""scripts/trace_persist.py -- per-phase timing of the persistent training kernel from its own %globaltimer stamps
(CTA 0's view): parameter fetch, images, epilogue + cluster reduce, owner gather, exchange/update/publish.
`--cluster=1` traces the variant without thread-block clusters.

    python scripts/trace_persist.py [B,B,...] [--cluster=1]
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pcnn_loader  # noqa: E402

pkg = pcnn_loader.load()
args = [x for x in sys.argv[1:] if not x.startswith("--")]
eng = pkg.Engine(0)
N = 262144
rng = np.random.default_rng(7)
eng.dataset_upload(pkg.TRAIN_SET, rng.integers(0, 256, (N, 784), dtype=np.uint8), rng.integers(0, 10, N, dtype=np.uint8))
eng.set_step_mode(pkg.MODE_PERSISTENT)
names = ["param_fetch", "images", "epilogue+cluster_reduce", "owner_gather", "update+publish"]
cl = [int(x.split("=")[1]) for x in sys.argv[1:] if x.startswith("--cluster=")]
if cl:
    eng.persist_tune(cl[0])
for B in [int(x) for x in (args[0].split(",") if args else ["1", "256", "1024"])]:
    eng.train_steps(0, B, 50)
    eng.persist_trace_arm()
    eng.train_steps(-1, B, 256)
    eng.sync()
    tr = eng.persist_trace_read(256)[8:]          # skip the first steps of the launch
    d = np.diff(tr, axis=1).astype(np.float64) / 1e3
    step = np.diff(tr[:, 0]).astype(np.float64) / 1e3
    row = {"kernel": "dataflow", "B": B, "step_us_median": float(np.median(step)),
           "next_step_gap_us": float(np.median(step) - np.median(d.sum(axis=1)))}
    row.update({n: float(np.median(d[:, i])) for i, n in enumerate(names)})
    row.update(eng.persist_info())
    print(json.dumps(row), flush=True)
eng.close()
