#!/usr/bin/env python
"""scripts/fcn_replica.py -- float32 torch CPU replicas of the segmenters FCNLite and FCNBilinear in tests/segment_nets.py
(test_segment_gpu's test_segmenter_trains): the same layers, initial masters, optimizer (SGD with momentum) and hyperparameters,
trained on the batches the device's ImageBatcher(pad=2, flip=True, masks=...) draws, replayed bit for bit by tests/augment_ref.py
(images) and tests/segment_ref.py (masks), against cross_entropy(ignore_index=255) with mean reduction; evaluated on the 256 golden
test digits with the running statistics.  Its test mIoU sets the end-to-end tests' thresholds.

Usage: fcn_replica.py [FCNLite] [FCNBilinear]"""
import sys

import numpy as np
import torch

import replica as R  # puts tests/ on the path
import augment_ref
import segment_nets
import segment_ref

F = torch.nn.functional
SEED, PAD = 5, 2                 # segment_nets.batchers: the training batcher's seed and padding


def miou(pred, target, O=segment_nets.O, ignore=segment_nets.IGNORE):
    """pkg.segmentation_scores' mIoU: IoU over the classes with a nonzero union, ignored targets left out"""
    keep = target != ignore
    t, p = target[keep].astype(np.int64), pred[keep].astype(np.int64)
    conf = np.bincount(t * O + p, minlength=O * O).reshape(O, O)
    tp = np.diag(conf).astype(np.float64)
    union = conf.sum(1) + conf.sum(0) - tp
    return float((tp[union > 0] / union[union > 0]).mean())


def batch_x(u8, first, N, shuffle, pad, flip, epoch):
    """the batcher's x: bf16 bits [N][28][28][8] (C_out 8, channels 1..7 zero) as float32 NCHW"""
    xb, *_ = augment_ref.batch(u8.reshape(-1, 28, 28, 1), first, N, shuffle, pad, flip, SEED, epoch, C_out=8)
    return torch.from_numpy((xb.astype(np.uint32) << 16).view(np.float32)).permute(0, 3, 1, 2).contiguous()


def run(name):
    cls = getattr(segment_nets, name)
    p = {k: torch.from_numpy(v) for k, v in cls.init_params().items()}
    w = {}
    for k, v in p.items():
        if k.startswith("f"):
            w[k] = v.permute(0, 3, 1, 2).contiguous()          # KRSC -> conv2d's [K][C][R][S]
        elif k == "w":
            w[k] = v.reshape(v.shape[0], -1)                    # [O][1][1][C] -> [O][C]
        else:
            w[k] = v.clone()                                    # t1, t2 already in ConvTranspose2d's [C_in][C_out][R][S]; bias
        w[k].requires_grad_(True)
    lite = name == "FCNLite"
    bn = R.bn_state((16, 32, 64, 32, 16) if lite else (16, 32, 64))
    b = lambda i, v, training: R.batch_norm(bn[i], v, training)

    def net(x, training):
        a = F.relu(b(0, F.conv2d(x, w["f1"], padding=1), training))
        bb = F.relu(b(1, F.conv2d(a, w["f2"], padding=1, stride=2), training))
        c = F.relu(b(2, F.conv2d(bb, w["f3"], padding=1, stride=2), training))
        if lite:
            d = F.relu(b(3, F.conv_transpose2d(c, w["t1"], stride=2, padding=1), training) + bb)
            e = F.relu(b(4, F.conv_transpose2d(d, w["t2"], stride=2, padding=1), training) + a)
            z = torch.einsum("nchw,oc->nhwo", e, w["w"]) + w["bw"]
        else:
            z7 = torch.einsum("nchw,oc->nohw", c, w["w"]) + w["bw"][None, :, None, None]
            z = F.interpolate(z7, size=(28, 28), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
        return z.reshape(-1, segment_nets.O)

    params = list(w.values()) + [t for ga, be, _, _ in bn for t in (ga, be)]
    opt = torch.optim.SGD(params, lr=cls.LR, momentum=cls.MOMENTUM)
    torch.manual_seed(0)
    g, *_ = R.golden()
    masks = segment_ref.digit_masks(g["train_u8"], g["train_labels"])
    test_masks = segment_ref.digit_masks(g["test_u8"], g["test_labels"])
    NB, steps = cls.NB, len(g["train_labels"]) // cls.NB
    losses = []
    for ep in range(cls.EPOCHS):
        for s in range(steps):
            x = batch_x(g["train_u8"], s * NB, NB, 1, PAD, 1, ep)
            m, *_ = segment_ref.mask_batch(masks, s * NB, NB, 1, PAD, 1, SEED, ep)
            loss = F.cross_entropy(net(x, True), torch.from_numpy(m.reshape(-1).astype(np.int64)), ignore_index=segment_nets.IGNORE)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(loss.item())
    preds = []
    with torch.no_grad():
        for s in range(len(g["test_labels"]) // NB):
            preds.append(net(batch_x(g["test_u8"], s * NB, NB, 0, 0, 0, 0), False).argmax(1).numpy())
    score = miou(np.concatenate(preds), test_masks[:len(preds) * NB].reshape(-1))
    print(f"{name}: mean loss epoch 1 {np.mean(losses[:steps]):.4f} -> epoch {cls.EPOCHS} {np.mean(losses[-steps:]):.4f}; "
          f"test mIoU {score:.4f}", flush=True)


if __name__ == "__main__":
    for name in sys.argv[1:] or ["FCNLite", "FCNBilinear"]:
        run(name)
