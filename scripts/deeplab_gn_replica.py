#!/usr/bin/env python
"""scripts/deeplab_gn_replica.py -- a float32 torch CPU replica of the segmenter DeepLabGN in tests/groupnorm_nets.py
(test_deeplab_gn_gpu's test_deeplab_gn_trains): the same layers, initial masters, optimizer (SGD with momentum) and hyperparameters,
trained on the batches the device's ImageBatcher(pad=2, flip=True, masks=...) draws (replayed by tests/augment_ref.py and
tests/segment_ref.py), against cross_entropy(ignore_index=255) with mean reduction; evaluated on the 256 golden test digits.  Its
test mIoU sets the end-to-end test's threshold.

--norm bn trains DeepLabLite's batch normalization instead (evaluated with the running statistics) at DeepLabGN's batch size and
hyperparameters, for comparison.  --lr and --epochs override the class's values (how they were chosen).

Usage: deeplab_gn_replica.py [--norm gn|bn] [--lr LR] [--epochs E]"""
import argparse

import numpy as np
import torch

import replica as R  # puts tests/ on the path
import fcn_replica
import groupnorm_nets
import segment_nets
import segment_ref

F = torch.nn.functional


def run(norm="gn", lr=None, epochs=None):
    cls = groupnorm_nets.DeepLabGN
    lr = cls.LR if lr is None else lr
    epochs = cls.EPOCHS if epochs is None else epochs
    torch.manual_seed(0)
    w = {}
    for k, v in cls.init_params().items():
        v = torch.from_numpy(v)
        if k == "wc":
            w[k] = v.reshape(32, 1, 3, 3).clone()               # [C][R][S] -> conv2d(groups=C)'s [C][1][R][S]
        elif k.startswith("f"):
            w[k] = v.permute(0, 3, 1, 2).contiguous()          # KRSC -> conv2d's [K][C][R][S]
        elif k == "w":
            w[k] = v.reshape(v.shape[0], -1)                    # [O][1][1][C] -> [O][C]
        else:
            w[k] = v.clone()
        w[k].requires_grad_(True)
    st = R.bn_state((16, 32, 32, 32, 32, 32, 32))
    if norm == "gn":
        b = lambda i, v, training: F.group_norm(v, cls.GROUPS, st[i][0], st[i][1], 1e-5)
    else:
        b = lambda i, v, training: R.batch_norm(st[i], v, training)

    def net(x, training):
        a = F.relu(b(0, F.conv2d(x, w["f1"], padding=1), training))
        bb = F.relu(b(1, F.conv2d(a, w["f2"], padding=1, stride=2), training))
        m = F.relu(b(2, F.conv2d(bb, w["fd1"], padding=2, dilation=2), training))
        h = F.relu(b(3, F.conv2d(m, w["fd2"], padding=2, dilation=2), training) + bb)
        sa = b(4, F.conv2d(m, w["fa"]), training)
        sb = b(5, F.conv2d(h, w["fb"], padding=4, dilation=4), training) + sa
        out = F.relu(b(6, F.conv2d(F.conv2d(h, w["wc"], padding=6, dilation=6, groups=32), w["fp"]), training) + sb)
        z14 = torch.einsum("nchw,oc->nohw", out, w["w"]) + w["bw"][None, :, None, None]
        z = F.interpolate(z14, size=(28, 28), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
        return z.reshape(-1, segment_nets.O)

    params = list(w.values()) + [t for ga, be, _, _ in st for t in (ga, be)]
    opt = torch.optim.SGD(params, lr=lr, momentum=cls.MOMENTUM)
    g, *_ = R.golden()
    masks = segment_ref.digit_masks(g["train_u8"], g["train_labels"])
    test_masks = segment_ref.digit_masks(g["test_u8"], g["test_labels"])
    NB, steps = cls.NB, len(g["train_labels"]) // cls.NB
    losses = []
    for ep in range(epochs):
        for s in range(steps):
            x = fcn_replica.batch_x(g["train_u8"], s * NB, NB, 1, fcn_replica.PAD, 1, ep)
            mk, *_ = segment_ref.mask_batch(masks, s * NB, NB, 1, fcn_replica.PAD, 1, fcn_replica.SEED, ep)
            loss = F.cross_entropy(net(x, True), torch.from_numpy(mk.reshape(-1).astype(np.int64)), ignore_index=segment_nets.IGNORE)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(loss.item())
    preds = []
    with torch.no_grad():
        for s in range(len(g["test_labels"]) // NB):
            preds.append(net(fcn_replica.batch_x(g["test_u8"], s * NB, NB, 0, 0, 0, 0), False).argmax(1).numpy())
    score = fcn_replica.miou(np.concatenate(preds), test_masks[:len(preds) * NB].reshape(-1))
    print(f"DeepLab{'GN' if norm == 'gn' else 'Lite'} at NB {NB}, lr {lr}, {epochs} epochs: mean loss epoch 1 "
          f"{np.mean(losses[:steps]):.4f} -> epoch {epochs} {np.mean(losses[-steps:]):.4f}; test mIoU {score:.4f}", flush=True)
    return score


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--norm", choices=("gn", "bn"), default="gn")
    ap.add_argument("--lr", type=float)
    ap.add_argument("--epochs", type=int)
    a = ap.parse_args()
    run(a.norm, a.lr, a.epochs)
