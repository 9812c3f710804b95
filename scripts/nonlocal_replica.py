#!/usr/bin/env python
"""scripts/nonlocal_replica.py -- float32 torch CPU replica of NonLocalResNet in tests/attention_nets.py (test_nonlocal_gpu's
test_nonlocal_resnet_mnist): the GAP ResNet of scripts/resnetgap_replica.py with a non-local block on its 12 x 12 x 16 activation
x1, x1n = BN(W_z softmax(q k^T / 4) v) + x1 with one head of 16 and the BN's gamma starting at 0; the same initialisation, batch
order (8 batches of 128 over the 1024 golden training digits per epoch), softmax cross-entropy over the batch and plain SGD,
evaluated on the 256 golden test digits with the running statistics.  Its accuracy sets the threshold of the end-to-end test.

Usage: nonlocal_replica.py [lr ...]"""
import argparse

import torch

import replica as R  # puts tests/ on the path
from attention_nets import NonLocalResNet

F = torch.nn.functional


def run(lr):
    net_cls = NonLocalResNet
    p = {k: torch.from_numpy(v) for k, v in net_cls.init_params().items()}
    w = {k: (p[k].permute(0, 3, 1, 2).contiguous() if k.startswith("f") else p[k].reshape(10, -1) if k == "w8" else p[k]).requires_grad_(True)
         for k in p}
    bn = R.bn_state((8, 16, 16, 16, 32, 32, 32, 16))
    with torch.no_grad():
        bn[7][0].zero_()                                   # the non-local block's BN: gamma 0
    b = lambda i, v, training: R.batch_norm(bn[i], v, training)
    d = net_cls.HEAD_DIM

    def nonlocal_block(x, training):
        B, C, H, W = x.shape
        t = x.permute(0, 2, 3, 1).reshape(B, H * W, C)
        q, k, v = F.linear(t, w["nl_wqkv"], w["nl_bqkv"]).split(d, -1)
        o = F.scaled_dot_product_attention(q[:, None], k[:, None], v[:, None])[:, 0]
        wz = F.linear(o, w["nl_wout"], w["nl_bout"]).reshape(B, H, W, C).permute(0, 3, 1, 2)
        return b(7, wz, training) + x

    def net(x, training):
        h = F.avg_pool2d(F.relu(b(0, F.conv2d(x, w["f1"]), training)), 2)
        x0 = F.relu(b(1, F.conv2d(h, w["f2"], padding=1), training))
        h = F.relu(b(2, F.conv2d(x0, w["f3"], padding=1), training))
        x1 = nonlocal_block(F.relu(b(3, F.conv2d(h, w["f4"], padding=1), training) + x0), training)
        h = F.relu(b(4, F.conv2d(x1, w["f5"], padding=1, stride=2), training))
        s = b(6, F.conv2d(x1, w["f7"], padding=1, stride=2), training)
        h = F.relu(b(5, F.conv2d(h, w["f6"], padding=1), training) + s)
        return F.linear(F.adaptive_avg_pool2d(h, 1).flatten(1), w["w8"], w["b8"])

    params = list(w.values()) + [t for ga, be, _, _ in bn for t in (ga, be)]
    R.run(net, params, lr, net_cls.EPOCHS, net_cls.NB, "sgd non-local ")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("lr", nargs="*", type=float)
    for lr in ap.parse_args().lr or [NonLocalResNet.LR_STEP]:
        run(lr)
