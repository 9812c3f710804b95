#!/usr/bin/env python
"""scripts/resnext_replica.py -- float32 torch CPU replica of the ResNeXt-style network of tests/test_gconv_gpu.py
(test_resnext_mnist): the same layers, initialisation, batch order (8 batches of 128 over the 1024 golden training digits per
epoch), softmax cross-entropy over the batch and plain SGD, evaluated on the 256 golden test digits with the running statistics.
Its accuracy sets the test's threshold.

Usage: resnext_replica.py [lr ...]"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
from test_gconv_gpu import EPOCHS, NB, init_params  # noqa: E402

F = torch.nn.functional


def run(lr):
    torch.manual_seed(0)
    g = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    img = lambda u8: torch.from_numpy(u8.reshape(-1, 1, 28, 28).astype(np.float32) / 255.0).bfloat16().float()   # the device's bf16 input
    xs, ys, xt, yt = img(g["train_u8"]), torch.from_numpy(g["train_labels"]).long(), img(g["test_u8"]), torch.from_numpy(g["test_labels"]).long()
    p = {k: torch.from_numpy(v) for k, v in init_params().items()}
    w = {k: (p[k].reshape(10, -1) if k == "w8" else p[k] if k == "b8" else p[k].permute(0, 3, 1, 2)).contiguous().requires_grad_(True)
         for k in p}
    bn = [(torch.ones(c, requires_grad=True), torch.zeros(c, requires_grad=True), torch.zeros(c), torch.ones(c))
          for c in (48, 64, 64, 48, 96, 96, 64)]

    def b(i, v, training):
        ga, be, rm, rv = bn[i]
        return F.batch_norm(v, rm, rv, ga, be, training=training, momentum=0.1, eps=1e-5)

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
    opt = torch.optim.SGD(params, lr=lr)
    losses = []
    for ep in range(EPOCHS):
        for s in range(1024 // NB):
            loss = F.cross_entropy(net(xs[s * NB:(s + 1) * NB], True), ys[s * NB:(s + 1) * NB])
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(loss.item())
    with torch.no_grad():
        acc = float((net(xt, False).argmax(1) == yt).float().mean())
    print(f"lr {lr}: mean loss epoch 1 {np.mean(losses[:8]):.4f} -> epoch {EPOCHS} {np.mean(losses[-8:]):.4f}; test accuracy {acc:.4f}",
          flush=True)


if __name__ == "__main__":
    for lr in [float(a) for a in sys.argv[1:]] or [0.2]:
        run(lr)
