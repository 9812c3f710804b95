#!/usr/bin/env python
"""scripts/efficientnet_replica.py -- float32 torch CPU replica of EfficientNetLite in tests/example_nets.py (test_bnact_gpu's
test_efficientnet_mnist): a SiLU stem, an MBConv with ReLU6, an MBConv with SiLU and squeeze-and-excitation carrying the residual,
and a hard-swish head; the same initialisation, batch order (8 batches of 128 over the 1024 golden training digits per epoch),
softmax cross-entropy over the batch and plain SGD, evaluated on the 256 golden test digits with the running statistics.  Its
accuracy sets the threshold of the end-to-end test.

Usage: efficientnet_replica.py [lr ...]"""
import argparse

import torch

import replica as R  # puts tests/ on the path
from example_nets import EfficientNetLite

F = torch.nn.functional


def masters(p):
    """the network's masters in torch's layouts, as leaves that take gradients"""
    conv = lambda k: torch.from_numpy(p[k]).permute(0, 3, 1, 2).contiguous().requires_grad_(True)         # KRSC -> KCRS
    dw = lambda k: torch.from_numpy(p[k]).unsqueeze(1).contiguous().requires_grad_(True)                   # [C][R][S] -> [C][1][R][S]
    w = {k: conv(k) for k in ("f0", "e1", "p1", "e2", "p2", "h")}
    w.update(d1=dw("d1"), d2=dw("d2"))
    w.update({k: torch.from_numpy(p[k].reshape(10, -1) if k == "w8" else p[k]).requires_grad_(True) for k in ("w8", "b8", "s1", "sb1", "s2", "sb2")})
    return w


def run(lr):
    w = masters(EfficientNetLite.init_params())
    bn = R.bn_state((48, 96, 96, 48, 96, 96, 48, 128))
    b = lambda i, v, training: R.batch_norm(bn[i], v, training)

    def net(x, training):
        h = F.avg_pool2d(F.silu(b(0, F.conv2d(x, w["f0"]), training)), 2)
        h = F.relu6(b(1, F.conv2d(h, w["e1"]), training))
        h = F.relu6(b(2, F.conv2d(h, w["d1"], stride=2, padding=1, groups=96), training))
        x1 = b(3, F.conv2d(h, w["p1"]), training)
        h = F.silu(b(4, F.conv2d(x1, w["e2"]), training))
        h = F.silu(b(5, F.conv2d(h, w["d2"], padding=2, groups=96), training))
        s = torch.sigmoid(F.linear(F.relu(F.linear(h.mean((2, 3)), w["s1"], w["sb1"])), w["s2"], w["sb2"]))
        h = h * s[:, :, None, None]
        x2 = b(6, F.conv2d(h, w["p2"]), training) + x1
        h = F.hardswish(b(7, F.conv2d(x2, w["h"]), training))
        return F.linear(F.adaptive_avg_pool2d(h, 1).flatten(1), w["w8"], w["b8"])

    params = list(w.values()) + [t for ga, be, _, _ in bn for t in (ga, be)]
    R.run(net, params, lr, EfficientNetLite.EPOCHS, EfficientNetLite.NB)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("lr", nargs="*", type=float)
    a = ap.parse_args()
    for lr in a.lr or [EfficientNetLite.LR_STEP]:
        run(lr)
