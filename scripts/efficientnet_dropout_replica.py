#!/usr/bin/env python
"""scripts/efficientnet_dropout_replica.py -- float32 torch CPU replica of EfficientNetDropout in tests/example_nets.py
(test_dropout_gpu's test_efficientnet_dropout_mnist): scripts/efficientnet_replica.py's network with element dropout (p = 0.2) on
the pooled features before the fc and stochastic depth (p = 0.2, per image) on the residual MBConv.  The masks are drawn from
tests/dropout_ref.py with the network's seeds and the layers' call counters (step k of training uses call k, from 1), so the
replica trains the same function as the device.  Its accuracy sets the threshold of the end-to-end test.

Usage: efficientnet_dropout_replica.py [lr ...]"""
import argparse
import itertools

import numpy as np
import torch

import replica as R  # puts tests/ on the path
import dropout_ref as D
from efficientnet_replica import masters
from example_nets import EfficientNetDropout

F = torch.nn.functional


def drop(p, seed, call, N, E, per_sample):
    """the multiplier m = kept ? fp32(1 / (1 - p)) : 0 of the device's mask, [N][E] (per image: [N][1])"""
    kept = D.keep(N, 1 if per_sample else E, p, seed, call, per_sample)
    return torch.from_numpy(np.where(kept, D.threshold(p)[1], np.float32(0)))


def run(lr):
    w = masters(EfficientNetDropout.init_params())
    bn = R.bn_state((48, 96, 96, 48, 96, 96, 48, 128))
    b = lambda i, v, training: R.batch_norm(bn[i], v, training)
    calls = itertools.count(1)                  # both layers count their training forwards, as DropoutLayer.call does

    def net(x, training):
        call = next(calls) if training else 0
        h = F.avg_pool2d(F.silu(b(0, F.conv2d(x, w["f0"]), training)), 2)
        h = F.relu6(b(1, F.conv2d(h, w["e1"]), training))
        h = F.relu6(b(2, F.conv2d(h, w["d1"], stride=2, padding=1, groups=96), training))
        x1 = b(3, F.conv2d(h, w["p1"]), training)
        h = F.silu(b(4, F.conv2d(x1, w["e2"]), training))
        h = F.silu(b(5, F.conv2d(h, w["d2"], padding=2, groups=96), training))
        s = torch.sigmoid(F.linear(F.relu(F.linear(h.mean((2, 3)), w["s1"], w["sb1"])), w["s2"], w["sb2"]))
        h = h * s[:, :, None, None]
        branch = b(6, F.conv2d(h, w["p2"]), training)
        if training:
            branch = branch * drop(EfficientNetDropout.P_PATH, EfficientNetDropout.SEED_PATH, call, x.shape[0], 0, True)[:, :, None, None]
        x2 = x1 + branch
        h = F.hardswish(b(7, F.conv2d(x2, w["h"]), training))
        feat = F.adaptive_avg_pool2d(h, 1).flatten(1)
        if training:
            feat = feat * drop(EfficientNetDropout.P_FC, EfficientNetDropout.SEED_FC, call, x.shape[0], feat.shape[1], False)
        return F.linear(feat, w["w8"], w["b8"])

    params = list(w.values()) + [t for ga, be, _, _ in bn for t in (ga, be)]
    R.run(net, params, lr, EfficientNetDropout.EPOCHS, EfficientNetDropout.NB)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("lr", nargs="*", type=float)
    a = ap.parse_args()
    for lr in a.lr or [EfficientNetDropout.LR_STEP]:
        run(lr)
