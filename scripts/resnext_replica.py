#!/usr/bin/env python
"""scripts/resnext_replica.py -- float32 torch CPU replica of ResNeXtLite in tests/example_nets.py (test_gconv_gpu's
test_resnext_mnist): the same layers, initialisation, batch order (8 batches of 128 over the 1024 golden training digits per
epoch), softmax cross-entropy over the batch and plain SGD, evaluated on the 256 golden test digits with the running statistics.
Its accuracy sets the test's threshold.

Usage: resnext_replica.py [lr ...]"""
import sys

import torch

import replica as R  # puts tests/ on the path
from example_nets import ResNeXtLite

F = torch.nn.functional


def run(lr):
    p = {k: torch.from_numpy(v) for k, v in ResNeXtLite.init_params().items()}
    w = {k: (p[k].reshape(10, -1) if k == "w8" else p[k] if k == "b8" else p[k].permute(0, 3, 1, 2)).contiguous().requires_grad_(True)
         for k in p}
    bn = R.bn_state((48, 64, 64, 48, 96, 96, 64))
    b = lambda i, v, training: R.batch_norm(bn[i], v, training)

    def net(x, training):
        x0 = F.relu(b(0, F.conv2d(x, w["f0"]), training))
        h = F.relu(b(1, F.conv2d(x0, w["e1"]), training))
        h = F.relu(b(2, F.conv2d(h, w["g1"], padding=1, groups=8), training))
        x1 = F.relu(b(3, F.conv2d(h, w["p1"]), training) + x0)
        h = F.relu(b(4, F.conv2d(x1, w["e2"]), training))
        h = F.relu(b(5, F.conv2d(h, w["g2"], stride=2, padding=1, groups=24), training))
        h = b(6, F.conv2d(h, w["p2"]), training)
        return F.linear(F.adaptive_avg_pool2d(h, 1).flatten(1), w["w8"], w["b8"])

    params = list(w.values()) + [t for ga, be, _, _ in bn for t in (ga, be)]
    R.run(net, params, lr, ResNeXtLite.EPOCHS, ResNeXtLite.NB, head="")


if __name__ == "__main__":
    for lr in [float(a) for a in sys.argv[1:]] or [0.2]:
        run(lr)
