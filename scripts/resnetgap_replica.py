#!/usr/bin/env python
"""scripts/resnetgap_replica.py -- float32 torch CPU replica of ResNetGAP in tests/example_nets.py (test_avgpool_nhwc_gpu's
test_resnet_gap_mnist): the same layers, initialisation, batch order (8 batches of 128 over the 1024 golden training digits per
epoch), softmax cross-entropy over the batch and an optimizer step, evaluated on the 256 golden test digits with the running
statistics.  Its accuracy sets the thresholds of the end-to-end tests.

Usage: resnetgap_replica.py [--optim sgd | momentum | adamw] [--augment | --mix | --resized | --trivial] [lr ...]
  sgd       plain SGD, p += -lr * grad (the layers' own sgd(lr); tests/test_avgpool_nhwc_gpu.py)
  momentum  torch.optim.SGD with momentum 0.9 and weight decay 5e-4 on every parameter (tests/test_optim_gpu.py)
  adamw     torch.optim.AdamW with betas (0.9, 0.999), eps 1e-8 and weight decay 1e-2 on every parameter (tests/test_optim_gpu.py)
  --augment each epoch's batches as pkg.ImageBatcher draws them with a shuffle and a random crop of pad 2, no flip, at the seed
            of tests/test_augment_gpu.py, replayed by tests/augment_ref.py (the device run: test_resnet_gap_through_the_batcher)
  --mix     --augment's batches mixed with MixUp (alpha 0.2) or CutMix (alpha 1.0) as the batcher draws them, against soft targets
            with label smoothing 0.1, replayed by tests/mix_ref.py (the device run: test_mix_gpu's test_resnet_gap_mixed)
  --resized each epoch's batches as pkg.ImageBatcher(crop_size=28, scale=(0.6, 1.0)) draws them with a shuffle, no flip,
            replayed by tests/resize_ref.py (the device run: test_resize_gpu's test_resnet_gap_on_resized_crops)
  --trivial --augment's batches with TrivialAugmentWide (BILINEAR) and RandomErasing(0.25) as pkg.ImageBatcher(trivial_augment=
            "bilinear", random_erase=0.25) draws them, replayed by tests/trivial_ref.py (the device run: test_trivial_gpu's
            test_resnet_gap_trivial_augmented)"""
import argparse

import torch

import replica as R  # puts tests/ on the path
from example_nets import ResNetGAP

F = torch.nn.functional


def run(lr, optim="sgd", augment=False, mix=False, resized=False, trivial=False):
    p = {k: torch.from_numpy(v) for k, v in ResNetGAP.init_params().items()}
    w = {k: (p[k].permute(0, 3, 1, 2).contiguous() if k.startswith("f") else p[k].reshape(10, -1) if k == "w8" else p[k]).requires_grad_(True)
         for k in p}
    bn = R.bn_state((8, 16, 16, 16, 32, 32, 32))
    b = lambda i, v, training: R.batch_norm(bn[i], v, training)

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
    head = f"{optim}{' mixed' if mix else ' augmented' if augment else ' resized' if resized else ' trivial' if trivial else ''} "
    R.run(net, params, lr, ResNetGAP.EPOCHS, ResNetGAP.NB, head, optim, augment, mix, resized, trivial)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--optim", default="sgd", choices=["sgd", "momentum", "adamw"])
    ap.add_argument("--augment", action="store_true")
    ap.add_argument("--mix", action="store_true")
    ap.add_argument("--resized", action="store_true")
    ap.add_argument("--trivial", action="store_true")
    ap.add_argument("lr", nargs="*", type=float)
    a = ap.parse_args()
    for lr in a.lr or [0.1]:
        run(lr, a.optim, a.augment, a.mix, a.resized, a.trivial)
