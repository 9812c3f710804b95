#!/usr/bin/env python
"""scripts/efficientnet_dropout_replica.py -- float32 torch CPU replica of the network of tests/test_dropout_gpu.py
(test_efficientnet_dropout_mnist): scripts/efficientnet_replica.py's network with element dropout (p = 0.2) on the pooled features
before the fc and stochastic depth (p = 0.2, per image) on the residual MBConv.  The masks are drawn from tests/dropout_ref.py with
the test's seeds and the layers' call counters (step k of training uses call k, from 1), so the replica trains the same function
as the device.  Its accuracy sets the threshold of the end-to-end test.

Usage: efficientnet_dropout_replica.py [lr ...]"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import dropout_ref as D  # noqa: E402
from test_bnact_gpu import EPOCHS, LR_STEP, NB, init_params  # noqa: E402
from test_dropout_gpu import P_FC, P_PATH, SEED_FC, SEED_PATH  # noqa: E402

F = torch.nn.functional


def drop(p, seed, call, N, E, per_sample):
    """the multiplier m = kept ? fp32(1 / (1 - p)) : 0 of the device's mask, [N][E] (per image: [N][1])"""
    kept = D.keep(N, 1 if per_sample else E, p, seed, call, per_sample)
    return torch.from_numpy(np.where(kept, D.threshold(p)[1], np.float32(0)))


def run(lr):
    torch.manual_seed(0)
    g = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    img = lambda u8: torch.from_numpy(u8.reshape(-1, 1, 28, 28).astype(np.float32) / 255.0).bfloat16().float()   # the device's bf16 input
    xs, ys, xt, yt = img(g["train_u8"]), torch.from_numpy(g["train_labels"]).long(), img(g["test_u8"]), torch.from_numpy(g["test_labels"]).long()
    p = init_params()
    conv = lambda k: torch.from_numpy(p[k]).permute(0, 3, 1, 2).contiguous().requires_grad_(True)         # KRSC -> KCRS
    dw = lambda k: torch.from_numpy(p[k]).unsqueeze(1).contiguous().requires_grad_(True)                   # [C][R][S] -> [C][1][R][S]
    w = {k: conv(k) for k in ("f0", "e1", "p1", "e2", "p2", "h")}
    w.update(d1=dw("d1"), d2=dw("d2"))
    w.update({k: torch.from_numpy(p[k].reshape(10, -1) if k == "w8" else p[k]).requires_grad_(True) for k in ("w8", "b8", "s1", "sb1", "s2", "sb2")})
    bn = [(torch.ones(c, requires_grad=True), torch.zeros(c, requires_grad=True), torch.zeros(c), torch.ones(c))
          for c in (48, 96, 96, 48, 96, 96, 48, 128)]

    def b(i, v, training):
        ga, be, rm, rv = bn[i]
        return F.batch_norm(v, rm, rv, ga, be, training=training, momentum=0.1, eps=1e-5)

    def net(x, training, call=0):
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
            branch = branch * drop(P_PATH, SEED_PATH, call, x.shape[0], 0, True)[:, :, None, None]
        x2 = x1 + branch
        h = F.hardswish(b(7, F.conv2d(x2, w["h"]), training))
        feat = F.adaptive_avg_pool2d(h, 1).flatten(1)
        if training:
            feat = feat * drop(P_FC, SEED_FC, call, x.shape[0], feat.shape[1], False)
        return F.linear(feat, w["w8"], w["b8"])

    params = list(w.values()) + [t for ga, be, _, _ in bn for t in (ga, be)]
    opt = torch.optim.SGD(params, lr=lr)
    losses = []
    call = 0
    for ep in range(EPOCHS):
        for s in range(1024 // NB):
            call += 1
            loss = F.cross_entropy(net(xs[s * NB:(s + 1) * NB], True, call), ys[s * NB:(s + 1) * NB])
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
    with torch.no_grad():
        acc = float((net(xt, False).argmax(1) == yt).float().mean())
    print(f"sgd lr {lr}: mean loss epoch 1 {np.mean(losses[:8]):.4f} -> epoch {EPOCHS} {np.mean(losses[-8:]):.4f}; test accuracy {acc:.4f}",
          flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("lr", nargs="*", type=float)
    a = ap.parse_args()
    for lr in a.lr or [LR_STEP]:
        run(lr)
