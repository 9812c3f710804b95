#!/usr/bin/env python
"""scripts/seresnet_replica.py -- float32 torch CPU replica of SEResNet in tests/example_nets.py (test_se_gpu's test_seresnet_mnist):
the GAP ResNet of scripts/resnetgap_replica.py with squeeze-and-excitation (16 -> 8 -> 16 and 32 -> 8 -> 32) carrying the residual
add and the ReLU of both blocks; the same initialisation, batch order (8 batches of 128 over the 1024 golden training digits per
epoch), softmax cross-entropy over the batch and plain SGD, evaluated on the 256 golden test digits with the running statistics.
Its accuracy sets the threshold of the end-to-end test.

Usage: seresnet_replica.py [lr ...]"""
import argparse

import torch

import replica as R  # puts tests/ on the path
from example_nets import SEResNet

F = torch.nn.functional


def run(lr):
    p = {k: torch.from_numpy(v) for k, v in SEResNet.init_params().items()}
    w = {k: (p[k].permute(0, 3, 1, 2).contiguous() if k.startswith("f") else p[k].reshape(10, -1) if k == "w8" else p[k]).requires_grad_(True)
         for k in p if not k.startswith("se")}
    se = {k: [p[f"{k}_{n}"].requires_grad_(True) for n in ("w1", "b1", "w2", "b2")] for k in ("se1", "se2")}
    bn = R.bn_state((8, 16, 16, 16, 32, 32, 32))
    b = lambda i, v, training: R.batch_norm(bn[i], v, training)

    def excite(k, v, r):
        w1, b1, w2, b2 = se[k]
        s = torch.sigmoid(F.linear(F.relu(F.linear(v.mean((2, 3)), w1, b1)), w2, b2))
        return F.relu(v * s[:, :, None, None] + r)

    def net(x, training):
        h = F.avg_pool2d(F.relu(b(0, F.conv2d(x, w["f1"]), training)), 2)
        x0 = F.relu(b(1, F.conv2d(h, w["f2"], padding=1), training))
        h = F.relu(b(2, F.conv2d(x0, w["f3"], padding=1), training))
        x1 = excite("se1", b(3, F.conv2d(h, w["f4"], padding=1), training), x0)
        h = F.relu(b(4, F.conv2d(x1, w["f5"], padding=1, stride=2), training))
        s = b(6, F.conv2d(x1, w["f7"], padding=1, stride=2), training)
        h = excite("se2", b(5, F.conv2d(h, w["f6"], padding=1), training), s)
        return F.linear(F.adaptive_avg_pool2d(h, 1).flatten(1), w["w8"], w["b8"])

    params = list(w.values()) + [t for ga, be, _, _ in bn for t in (ga, be)] + [t for v in se.values() for t in v]
    R.run(net, params, lr, SEResNet.EPOCHS, SEResNet.NB)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("lr", nargs="*", type=float)
    a = ap.parse_args()
    for lr in a.lr or [0.2]:
        run(lr)
