#!/usr/bin/env python
"""scripts/seresnet_replica.py -- float32 torch CPU replica of the SE-ResNet of tests/test_se_gpu.py (test_seresnet_mnist): the
GAP ResNet of scripts/resnetgap_replica.py with squeeze-and-excitation (16 -> 8 -> 16 and 32 -> 8 -> 32) carrying the residual add
and the ReLU of both blocks; the same initialisation, batch order (8 batches of 128 over the 1024 golden training digits per
epoch), softmax cross-entropy over the batch and plain SGD, evaluated on the 256 golden test digits with the running statistics.
Its accuracy sets the threshold of the end-to-end test.

Usage: seresnet_replica.py [lr ...]"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_avgpool_nhwc_gpu import NB, init_params  # noqa: E402
from test_se_gpu import EPOCHS, init_se  # noqa: E402

F = torch.nn.functional


def run(lr):
    torch.manual_seed(0)
    g = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    img = lambda u8: torch.from_numpy(u8.reshape(-1, 1, 28, 28).astype(np.float32) / 255.0).bfloat16().float()   # the device's bf16 input
    xs, ys, xt, yt = img(g["train_u8"]), torch.from_numpy(g["train_labels"]).long(), img(g["test_u8"]), torch.from_numpy(g["test_labels"]).long()
    p = {k: torch.from_numpy(v) for k, v in init_params().items()}
    w = {k: (p[k].permute(0, 3, 1, 2).contiguous() if k.startswith("f") else p[k].reshape(10, -1) if k == "w8" else p[k]).requires_grad_(True)
         for k in p}
    se = {k: [torch.from_numpy(a.copy()).requires_grad_(True) for a in v] for k, v in init_se().items()}
    bn = [(torch.ones(c, requires_grad=True), torch.zeros(c, requires_grad=True), torch.zeros(c), torch.ones(c)) for c in (8, 16, 16, 16, 32, 32, 32)]

    def b(i, v, training):
        ga, be, rm, rv = bn[i]
        return F.batch_norm(v, rm, rv, ga, be, training=training, momentum=0.1, eps=1e-5)

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
    opt = torch.optim.SGD(params, lr=lr)
    losses = []
    for ep in range(EPOCHS):
        for s in range(1024 // NB):
            loss = F.cross_entropy(net(xs[s * NB:(s + 1) * NB], True), ys[s * NB:(s + 1) * NB])
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(float(loss))
    with torch.no_grad():
        acc = float((net(xt, False).argmax(1) == yt).float().mean())
    print(f"sgd lr {lr}: mean loss epoch 1 {np.mean(losses[:8]):.4f} -> epoch {EPOCHS} {np.mean(losses[-8:]):.4f}; test accuracy {acc:.4f}",
          flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("lr", nargs="*", type=float)
    a = ap.parse_args()
    for lr in a.lr or [0.2]:
        run(lr)
