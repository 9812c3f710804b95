#!/usr/bin/env python
"""scripts/vae_replica.py -- a float32 torch CPU replica of ConvVAE in tests/vae_nets.py (test_vae_nets_gpu): the same layers,
initial masters, optimizer (AdamW, torch's defaults but the learning rate) and hyperparameters, trained on the batches the device's
ImageBatcher(pad=2, flip=True) draws (replayed by tests/augment_ref.py), with the latent's eps drawn by tests/vae_ref.py from the
device layers' seeds and calls, so the two runs differ only by arithmetic.  Prints the test negative ELBO per image in nats, its
reconstruction and KL parts, and the mean-image baseline's; its ELBO sets the end-to-end test's threshold."""
import numpy as np
import torch

import replica as R  # puts tests/ on the path
import vae_nets
import vae_ref
from restore_replica import PAD, batch_x

F = torch.nn.functional


def run():
    cls = vae_nets.ConvVAE
    B, L, beta = cls.NB, cls.L, cls.BETA
    w = {}
    for k, v in cls.init_params().items():
        v = torch.from_numpy(v)
        if k in ("f1", "f2"):
            v = v.permute(0, 3, 1, 2).contiguous()                  # KRSC -> conv2d's [K][C][R][S]
        elif k == "we":
            v = v.reshape(2 * L, -1)                                 # [O][7][7][64]: NHWC flattening, as the device reads y2
        elif k in ("wd", "w"):
            v = v.reshape(v.shape[0], -1)
        w[k] = v.clone().requires_grad_(True)

    def net(x, eps):
        h = F.relu(F.conv2d(x, w["f1"], w["b1"], stride=2, padding=1))
        h = F.relu(F.conv2d(h, w["f2"], w["b2"], stride=2, padding=1))
        st = h.permute(0, 2, 3, 1).reshape(B, -1) @ w["we"].t() + w["be"]
        mu, lv = st[:, :L], st[:, L:]
        z = mu + torch.exp(0.5 * lv) * eps
        kl = 0.5 * (mu * mu + torch.exp(lv) - 1 - lv).sum(1)
        d = F.relu(z @ w["wd"].t() + w["bd"]).reshape(B, 4, 4, 16).permute(0, 3, 1, 2)      # a dense 4 x 4 x 16 NHWC map
        d = F.relu(F.conv_transpose2d(d, w["t1"], w["tb1"], stride=2, padding=1))
        d = F.relu(F.conv_transpose2d(d, w["t2"], w["tb2"], stride=2, padding=1, output_padding=1))
        o = torch.einsum("nchw,oc->nohw", d, w["w"]) + w["bw"][None, :, None, None]
        logits = F.pixel_shuffle(o, 2)
        rec = F.binary_cross_entropy_with_logits(logits, x[:, :1], reduction="none").reshape(B, -1).sum(1)
        return rec, kl

    opt = torch.optim.AdamW(list(w.values()), lr=cls.LR)
    torch.manual_seed(0)
    g, *_ = R.golden()
    steps = len(g["train_labels"]) // B
    losses, call = [], 0
    for ep in range(cls.EPOCHS):
        for s in range(steps):
            x = batch_x(g["train_u8"], s * B, B, 1, PAD, 1, ep)
            call += 1
            rec, kl = net(x, torch.from_numpy(vae_ref.eps(B, L, cls.SEED_LATENT, call)))
            loss = (rec + beta * kl).mean()
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(loss.item())
    recs, kls, x0 = [], [], []
    with torch.no_grad():
        for s in range(len(g["test_labels"]) // B):
            x = batch_x(g["test_u8"], s * B, B, 0, 0, 0, 0)
            rec, kl = net(x, torch.from_numpy(vae_ref.eps(B, L, cls.SEED_TEST_LATENT, s + 1)))
            recs.append(rec)
            kls.append(kl)
            x0.append(x[:, 0].numpy())
    rec, kl = torch.cat(recs).double().mean().item(), torch.cat(kls).double().mean().item()
    base = vae_nets.mean_image_nelbo(g, np.concatenate(x0))
    print(f"ConvVAE: mean loss epoch 1 {np.mean(losses[:steps]):.2f} -> epoch {cls.EPOCHS} {np.mean(losses[-steps:]):.2f}; test "
          f"negative ELBO {rec + kl:.2f} nats (reconstruction {rec:.2f}, KL {kl:.2f}), mean-image baseline {base:.2f}", flush=True)


if __name__ == "__main__":
    run()
