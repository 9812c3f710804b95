#!/usr/bin/env python
"""scripts/resnetgap_replica.py -- float32 torch CPU replica of the GAP ResNet of tests/test_avgpool_nhwc_gpu.py
(test_resnet_gap_mnist): the same layers, initialisation, batch order (8 batches of 128 over the 1024 golden training digits per
epoch), softmax cross-entropy over the batch and an optimizer step, evaluated on the 256 golden test digits with the running
statistics.  Its accuracy sets the thresholds of the end-to-end tests.

Usage: resnetgap_replica.py [--optim sgd | momentum | adamw] [--augment] [lr ...]
  sgd       plain SGD, p += -lr * grad (the layers' own sgd(lr); tests/test_avgpool_nhwc_gpu.py)
  momentum  torch.optim.SGD with momentum 0.9 and weight decay 5e-4 on every parameter (tests/test_optim_gpu.py)
  adamw     torch.optim.AdamW with betas (0.9, 0.999), eps 1e-8 and weight decay 1e-2 on every parameter (tests/test_optim_gpu.py)
  --augment each epoch's batches as pkg.ImageBatcher draws them with a shuffle and a random crop of pad 2, no flip, at the seed
            of tests/test_augment_gpu.py, replayed by tests/augment_ref.py (the device run: test_resnet_gap_through_the_batcher)"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_avgpool_nhwc_gpu import EPOCHS, NB, init_params  # noqa: E402

AUG_SEED, AUG_PAD = 0x0123456789ABCDEF, 2       # tests/test_augment_gpu.py

F = torch.nn.functional


def run(lr, optim="sgd", augment=False):
    torch.manual_seed(0)
    g = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    img = lambda u8: torch.from_numpy(u8.reshape(-1, 1, 28, 28).astype(np.float32) / 255.0).bfloat16().float()   # the device's bf16 input
    xs, ys, xt, yt = img(g["train_u8"]), torch.from_numpy(g["train_labels"]).long(), img(g["test_u8"]), torch.from_numpy(g["test_labels"]).long()
    p = {k: torch.from_numpy(v) for k, v in init_params().items()}
    w = {k: (p[k].permute(0, 3, 1, 2).contiguous() if k.startswith("f") else p[k].reshape(10, -1) if k == "w8" else p[k]).requires_grad_(True)
         for k in p}
    bn = [(torch.ones(c, requires_grad=True), torch.zeros(c, requires_grad=True), torch.zeros(c), torch.ones(c)) for c in (8, 16, 16, 16, 32, 32, 32)]

    def b(i, v, training):
        ga, be, rm, rv = bn[i]
        return F.batch_norm(v, rm, rv, ga, be, training=training, momentum=0.1, eps=1e-5)

    def net(x, training):
        h = F.avg_pool2d(F.relu(b(0, F.conv2d(x, w["f1"]), training)), 2)
        x0 = F.relu(b(1, F.conv2d(h, w["f2"], padding=1), training))
        h = F.relu(b(2, F.conv2d(x0, w["f3"], padding=1), training))
        x1 = F.relu(b(3, F.conv2d(h, w["f4"], padding=1), training) + x0)
        h = F.relu(b(4, F.conv2d(x1, w["f5"], padding=1, stride=2), training))
        s = b(6, F.conv2d(x1, w["f7"], padding=1, stride=2), training)
        h = F.relu(b(5, F.conv2d(h, w["f6"], padding=1), training) + s)
        return F.linear(F.adaptive_avg_pool2d(h, 1).flatten(1), w["w8"], w["b8"])

    params = list(w.values()) + [t for ga, be, _, _ in bn for t in (ga, be)]
    opt = {"sgd": lambda: torch.optim.SGD(params, lr=lr),
           "momentum": lambda: torch.optim.SGD(params, lr=lr, momentum=0.9, weight_decay=5e-4),
           "adamw": lambda: torch.optim.AdamW(params, lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)}[optim]()
    losses = []
    for ep in range(EPOCHS):
        for s in range(1024 // NB):
            if augment:
                import augment_ref
                xb, lab, *_ = augment_ref.batch(g["train_u8"].reshape(-1, 28, 28, 1), s * NB, NB, 1, AUG_PAD, 0, AUG_SEED, ep,
                                                labels=g["train_labels"])
                x = torch.from_numpy((xb.astype(np.uint32) << 16).view(np.float32).reshape(NB, 1, 28, 28))
                loss = F.cross_entropy(net(x, True), torch.from_numpy(lab).long())
            else:
                loss = F.cross_entropy(net(xs[s * NB:(s + 1) * NB], True), ys[s * NB:(s + 1) * NB])
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(float(loss))
    with torch.no_grad():
        acc = float((net(xt, False).argmax(1) == yt).float().mean())
    print(f"{optim}{' augmented' if augment else ''} lr {lr}: mean loss epoch 1 {np.mean(losses[:8]):.4f} -> epoch {EPOCHS} {np.mean(losses[-8:]):.4f}; test accuracy {acc:.4f}",
          flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--optim", default="sgd", choices=["sgd", "momentum", "adamw"])
    ap.add_argument("--augment", action="store_true")
    ap.add_argument("lr", nargs="*", type=float)
    a = ap.parse_args()
    for lr in a.lr or [0.1]:
        run(lr, a.optim, a.augment)
