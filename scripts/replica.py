"""What the float32 torch CPU replicas of the example networks (tests/example_nets.py) share: the golden digits as the device sees
them, the batch-norm state, and the loop that trains a replica's net on them and prints its line.  A replica supplies its net,
the layout of its masters and its options; it needs torch and numpy, not the package."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
F = torch.nn.functional
AUG_SEED, AUG_PAD = 0x0123456789ABCDEF, 2       # tests/test_augment_gpu.py
MIX_ALPHAS, MIX_EPS = (0.2, 1.0), 0.1           # tests/test_mix_gpu.py: mixup_alpha, cutmix_alpha and label smoothing
DIGIT_SCALE = (0.6, 1.0)                        # tests/test_resize_gpu.py: RandomResizedCrop(28, scale) of the digits
TRIVIAL_ERASE = 0.25                            # tests/test_trivial_gpu.py: TrivialAugmentWide (BILINEAR) and RandomErasing(p)


def golden():
    """the golden subset, and its training and test digits as [n][1][28][28] float32 holding the device's bf16 input, with labels"""
    g = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    img = lambda u8: torch.from_numpy(u8.reshape(-1, 1, 28, 28).astype(np.float32) / 255.0).bfloat16().float()
    return g, img(g["train_u8"]), torch.from_numpy(g["train_labels"]).long(), img(g["test_u8"]), torch.from_numpy(g["test_labels"]).long()


def bn_state(channels):
    """(gamma, beta, running mean, running var) of each batch norm, as a fresh BatchNormLayer starts"""
    return [(torch.ones(c, requires_grad=True), torch.zeros(c, requires_grad=True), torch.zeros(c), torch.ones(c)) for c in channels]


def batch_norm(state, v, training):
    ga, be, rm, rv = state
    return F.batch_norm(v, rm, rv, ga, be, training=training, momentum=0.1, eps=1e-5)


def run(net, params, lr, epochs, NB, head="sgd ", optim="sgd", augment=False, mix=False, resized=False, trivial=False):
    """net(x, training) trained for `epochs` epochs of the 1024 golden training digits in order, NB per batch, with softmax
    cross-entropy over the batch and an optimizer step on params, then evaluated on the 256 golden test digits; prints the mean
    loss of the first and last epoch and the accuracy after `head`.
      optim    sgd: plain SGD (the layers' own sgd(lr)); momentum: torch.optim.SGD with momentum 0.9 and weight decay 5e-4;
               adamw: torch.optim.AdamW with betas (0.9, 0.999), eps 1e-8 and weight decay 1e-2
      augment  each epoch's batches as pkg.ImageBatcher draws them with a shuffle and a random crop of pad 2, no flip, at the seed
               of tests/test_augment_gpu.py, replayed by tests/augment_ref.py
      mix      augment's batches, each mixed as an ImageBatcher with MIX_ALPHAS mixes it (tests/mix_ref.py), trained against
               the soft target of pcnn_softmax_ce_soft_bf16 with label smoothing MIX_EPS
      resized  each epoch's batches as an ImageBatcher with crop_size 28 and scale DIGIT_SCALE draws them (shuffle, no flip),
               replayed by tests/resize_ref.py; the test digits go through Resize(28) + CenterCrop(28), which leaves them as they are
      trivial  augment's batches with TrivialAugmentWide (BILINEAR) after the crop and RandomErasing(TRIVIAL_ERASE) after
               Normalize, as an ImageBatcher(trivial_augment="bilinear", random_erase=TRIVIAL_ERASE) draws them, replayed by
               tests/trivial_ref.py"""
    torch.manual_seed(0)
    g, xs, ys, xt, yt = golden()
    opt = {"sgd": lambda: torch.optim.SGD(params, lr=lr),
           "momentum": lambda: torch.optim.SGD(params, lr=lr, momentum=0.9, weight_decay=5e-4),
           "adamw": lambda: torch.optim.AdamW(params, lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)}[optim]()
    steps = len(ys) // NB
    losses = []
    if trivial:
        import trivial_ref
        tab28 = trivial_ref.table(28, 28)
    for ep in range(epochs):
        for s in range(steps):
            if mix:
                import mix_ref
                kind, _, box, lam, _ = mix_ref.draws(AUG_SEED, ep, s, 28, 28, *MIX_ALPHAS)
                mode = mix_ref.MIXUP if kind == "mixup" else mix_ref.CUTMIX
                xb, lab, lab_b = mix_ref.batch(g["train_u8"].reshape(-1, 28, 28, 1), s * NB, NB, mode, lam, box or (0, 0, 0, 0), 1,
                                               AUG_PAD, 0, AUG_SEED, ep, labels=g["train_labels"])
                x = torch.from_numpy((xb.astype(np.uint32) << 16).view(np.float32).reshape(NB, 1, 28, 28))
                y = torch.from_numpy(mix_ref.soft_target(lab, lab_b, lam, MIX_EPS, 10)[1])
            elif trivial:
                xb, lab, *_ = trivial_ref.batch(g["train_u8"].reshape(-1, 28, 28, 1), s * NB, NB, trivial_ref.BILINEAR, TRIVIAL_ERASE,
                                                pad=AUG_PAD, seed=AUG_SEED, epoch=ep, labels=g["train_labels"], tab=tab28)
                x, y = torch.from_numpy((xb.astype(np.uint32) << 16).view(np.float32).reshape(NB, 1, 28, 28)), torch.from_numpy(lab).long()
            elif resized:
                import resize_ref
                xb, lab, *_ = resize_ref.batch(g["train_u8"].reshape(-1, 28, 28, 1), s * NB, NB, resize_ref.TRAIN, 28, 28, DIGIT_SCALE,
                                               seed=AUG_SEED, epoch=ep, labels=g["train_labels"])
                x, y = torch.from_numpy((xb.astype(np.uint32) << 16).view(np.float32).reshape(NB, 1, 28, 28)), torch.from_numpy(lab).long()
            elif augment:
                import augment_ref
                xb, lab, *_ = augment_ref.batch(g["train_u8"].reshape(-1, 28, 28, 1), s * NB, NB, 1, AUG_PAD, 0, AUG_SEED, ep,
                                                labels=g["train_labels"])
                x, y = torch.from_numpy((xb.astype(np.uint32) << 16).view(np.float32).reshape(NB, 1, 28, 28)), torch.from_numpy(lab).long()
            else:
                x, y = xs[s * NB:(s + 1) * NB], ys[s * NB:(s + 1) * NB]
            loss = F.cross_entropy(net(x, True), y)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(loss.item())
    with torch.no_grad():
        acc = float((net(xt, False).argmax(1) == yt).float().mean())
    print(f"{head}lr {lr}: mean loss epoch 1 {np.mean(losses[:steps]):.4f} -> epoch {epochs} {np.mean(losses[-steps:]):.4f}; "
          f"test accuracy {acc:.4f}", flush=True)
