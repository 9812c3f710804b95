#!/usr/bin/env python
"""scripts/deeplab_replica.py -- a float32 torch CPU replica of the segmenter DeepLabLite in tests/deeplab_nets.py
(test_deeplab_gpu's test_deeplab_trains): the same layers, initial masters, optimizer (SGD with momentum) and hyperparameters,
trained on the batches the device's ImageBatcher(pad=2, flip=True, masks=...) draws (replayed by tests/augment_ref.py and
tests/segment_ref.py), against cross_entropy(ignore_index=255) with mean reduction; evaluated on the 256 golden test digits with
the running statistics.  Its test mIoU sets the end-to-end test's threshold.

Usage: deeplab_replica.py"""
import numpy as np
import torch

import replica as R  # puts tests/ on the path
import deeplab_nets
import fcn_replica
import segment_nets
import segment_ref

F = torch.nn.functional


def run():
    cls = deeplab_nets.DeepLabLite
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
    bn = R.bn_state((16, 32, 32, 32, 32, 32, 32))
    b = lambda i, v, training: R.batch_norm(bn[i], v, training)

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
    print(f"DeepLabLite: mean loss epoch 1 {np.mean(losses[:steps]):.4f} -> epoch {cls.EPOCHS} {np.mean(losses[-steps:]):.4f}; "
          f"test mIoU {score:.4f}", flush=True)


if __name__ == "__main__":
    run()
