#!/usr/bin/env python
"""scripts/restore_replica.py -- float32 torch CPU replicas of the restorers ESPCNLite and DenoiseNet in tests/restore_nets.py
(test_restore_nets_gpu): the same layers, initial masters, optimizer (AdamW, torch's defaults but the learning rate) and
hyperparameters, trained on the batches the device's ImageBatcher(pad=2, flip=True) draws, replayed bit for bit by
tests/augment_ref.py, with DenoiseNet's masking noise drawn by tests/dropout_ref.py from the device layer's seeds and calls.  Evaluated
on the 256 golden test digits with the running statistics; prints the test PSNR and the baseline's.  Its PSNR sets the end-to-end
tests' thresholds.

Usage: restore_replica.py [ESPCNLite] [DenoiseNet]"""
import sys

import numpy as np
import torch

import replica as R  # puts tests/ on the path
import augment_ref
import dropout_ref
import restore_nets

F = torch.nn.functional
SEED, PAD = 5, 2                 # restore_nets.batchers: the training batcher's seed and padding


def psnr(pred, target):
    """pkg.psnr: the mean over images of 10 log10(1 / MSE) in float64"""
    mse = ((pred.double() - target.double()) ** 2).reshape(len(pred), -1).mean(1)
    return float((10 * torch.log10(1.0 / mse)).mean())


def batch_x(u8, first, N, shuffle, pad, flip, epoch):
    """the batcher's x: bf16 bits [N][28][28][8] (channels 1..7 zero) as float32 NCHW"""
    xb, *_ = augment_ref.batch(u8.reshape(-1, 28, 28, 1), first, N, shuffle, pad, flip, SEED, epoch, C_out=8)
    return torch.from_numpy((xb.astype(np.uint32) << 16).view(np.float32)).permute(0, 3, 1, 2).contiguous()


def corrupt(x, seed, call, p):
    """DropoutLayer's forward on x (NCHW float32 of bf16 values): the Philox mask of (seed, call) over the NHWC rows, bf16 values"""
    N = x.shape[0]
    xh = x.permute(0, 2, 3, 1).reshape(N, -1).numpy()
    y, _ = dropout_ref.dropout(xh, p, seed, call)
    return torch.from_numpy(np.ascontiguousarray(y)).reshape(N, 28, 28, 8).permute(0, 3, 1, 2).contiguous()


def run(name):
    cls = getattr(restore_nets, name)
    p = {k: torch.from_numpy(v) for k, v in cls.init_params().items()}
    w = {}
    for k, v in p.items():
        if k.startswith("f"):
            w[k] = v.permute(0, 3, 1, 2).contiguous()          # KRSC -> conv2d's [K][C][R][S]
        elif k == "w":
            w[k] = v.reshape(v.shape[0], -1)                    # [O][1][1][C] -> [O][C]
        else:
            w[k] = v.clone()
        w[k].requires_grad_(True)
    espcn = name == "ESPCNLite"
    bn = [] if espcn else R.bn_state((16, 64))

    def head(h):
        z = torch.einsum("nchw,oc->nohw", h, w["w"]) + w["bw"][None, :, None, None]
        return F.pixel_shuffle(z, 2)

    def net(x, training):
        if espcn:
            lr = F.avg_pool2d(x, 2)
            h = F.relu(F.conv2d(lr, w["f1"], w["b1"], padding=2))
            return head(F.relu(F.conv2d(h, w["f2"], w["b2"], padding=1))), F.interpolate(lr, scale_factor=2, mode="bilinear",
                                                                                         align_corners=False)
        h = F.relu(R.batch_norm(bn[0], F.conv2d(x, w["f1"], padding=1), training))
        h = F.relu(R.batch_norm(bn[1], F.conv2d(F.pixel_unshuffle(h, 2), w["f2"], padding=1), training))
        return head(h), x

    params = list(w.values()) + [t for ga, be, _, _ in bn for t in (ga, be)]
    opt = torch.optim.AdamW(params, lr=cls.LR)
    loss_fn = F.mse_loss if espcn else F.l1_loss
    torch.manual_seed(0)
    g, *_ = R.golden()
    NB, steps = cls.NB, len(g["train_labels"]) // cls.NB
    losses, call = [], 0
    for ep in range(cls.EPOCHS):
        for s in range(steps):
            x = batch_x(g["train_u8"], s * NB, NB, 1, PAD, 1, ep)
            xin = x
            if not espcn:
                call += 1
                xin = corrupt(x, cls.SEED_NOISE, call, cls.P_NOISE)
            loss = loss_fn(net(xin, True)[0], x[:, :1])
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(loss.item())
    preds, base, clean = [], [], []
    with torch.no_grad():
        for s in range(len(g["test_labels"]) // NB):
            x = batch_x(g["test_u8"], s * NB, NB, 0, 0, 0, 0)
            xin = x if espcn else corrupt(x, cls.SEED_TEST_NOISE, s + 1, cls.P_NOISE)
            out, bl = net(xin, False)
            preds.append(out[:, 0])
            base.append(bl[:, 0])
            clean.append(x[:, 0])
    clean = torch.cat(clean)
    print(f"{name}: mean loss epoch 1 {np.mean(losses[:steps]):.5f} -> epoch {cls.EPOCHS} {np.mean(losses[-steps:]):.5f}; "
          f"test PSNR {psnr(torch.cat(preds), clean):.2f} dB, baseline {psnr(torch.cat(base), clean):.2f} dB", flush=True)


if __name__ == "__main__":
    for name in sys.argv[1:] or ["ESPCNLite", "DenoiseNet"]:
        run(name)
