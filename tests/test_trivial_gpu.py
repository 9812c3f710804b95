"""TrivialAugmentWide and RandomErasing on the device (pcnn_augment_trivial_u8_bf16, ImageBatcher(trivial_augment=..., random_erase=...)):
x and labels bit for bit against trivial_ref's replay in both interpolations, with and without erasing, over MNIST in the [28][32]
layout, CIFAR-sized crops into C_out 3 and 8, 256 -> 224 RandomResizedCrop at N = 256 and a pitched odd shape, with every op drawn
at many bins; torchvision's _apply_op + Normalize on the device's own draws; reruns, batch sizes that split an epoch differently,
untouched pads and tails, refusals, and the batcher."""
import numpy as np
import pytest
import torch
from torchvision.transforms import InterpolationMode
from torchvision.transforms import autoaugment as aa

import augment_ref as A
import trivial_ref as TR
from example_nets import DEV, NAN_BF16
from example_nets import ResNetGAP, train
from test_augment_gpu import CIFAR, IMAGENET, LABEL_SENTINEL, SEED, TAIL, bits, dev, synthetic, x_buffer
from test_trivial_cpu import neighbours

pytestmark = pytest.mark.gpu


def run_case(eng, pkg, images, labels, first, N, trivial, erase_p, crop_size=None, pad=0, flip=1, epoch=0, mean=None, std=None,
             C_out=None, row_pitch=0, image_rows=0, shuffle=1):
    """one call on fresh NaN-filled buffers: (x [N][h][w][C_out] bits, labels_out) after checking pads and tails"""
    n, H, W, C = images.shape
    C_out = C if C_out is None else C_out
    info = pkg.augment_trivial_info(n, H, W, C, first, N, trivial, erase_p, crop_size=crop_size, shuffle=shuffle, pad=pad, flip=flip,
                                    C_out=C_out, row_pitch=row_pitch, image_rows=image_rows, mean=mean, std=std)[0]
    rows, pitch, h, w = info["image_rows"], info["row_pitch"], info["h"], info["w"]
    x = x_buffer(N, rows, pitch)
    ws = torch.full((info["ws_bytes"],), 0x5A, dtype=torch.uint8, device=DEV)
    lo = None if labels is None else torch.full((N + TAIL,), LABEL_SENTINEL, dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()                              # the engine's stream does not wait for torch's fills
    eng.augment_trivial(images, labels, n, H, W, C, first, N, x, ws, lo, trivial=trivial, erase_p=erase_p, crop_size=crop_size,
                        shuffle=shuffle, pad=pad, flip=flip, seed=SEED, epoch=epoch, mean=mean, std=std, C_out=C_out, row_pitch=row_pitch,
                        image_rows=image_rows)
    eng.sync()
    xb = bits(x)
    assert (xb[N * rows * pitch:] == NAN_BF16).all()                      # past x
    xb = xb[:N * rows * pitch].reshape(N, rows, pitch)
    assert (xb[:, :, w * C_out:] == NAN_BF16).all() and (xb[:, h:, :] == NAN_BF16).all()
    lob = None
    if lo is not None:
        lob = lo.cpu().numpy()
        assert (lob[N:] == LABEL_SENTINEL).all()
        lob = lob[:N]
    return xb[:, :h, :w * C_out].reshape(N, h, w, C_out), lob


CASES = {  # name: (dataset (n, H, W, C) or "mnist", first, N, crop_size, pad, epoch, mean, std, C_out, row_pitch, image_rows)
    "mnist-28x32-pad2": ("mnist", 128, 128, None, 2, 3, None, None, 1, 32, 28),
    "cifar-pad4-cout3": ((1024, 32, 32, 3), 256, 256, None, 4, 1, *CIFAR, 3, 0, 0),
    "cifar-pad4-cout8": ((1024, 32, 32, 3), 256, 256, None, 4, 2, *CIFAR, 8, 0, 0),
    "odd-pitched": ((100, 27, 45, 3), 3, 17, None, 3, 5, (0.3, 0.1, 0.2), (0.7, 0.2, 0.4), 5, 232, 30),
    "imagenet-256-224": ((300, 256, 256, 3), 32, 256, (224, 224), 0, 1, *IMAGENET, 8, 0, 0),
}


def dataset(golden, spec):
    if spec == "mnist":
        return golden["train_u8"].reshape(-1, 28, 28, 1), golden["train_labels"]
    return synthetic(*spec)


@pytest.mark.parametrize("erase_p", [0.0, 0.5])
@pytest.mark.parametrize("trivial", [TR.NEAREST, TR.BILINEAR])
@pytest.mark.parametrize("name", list(CASES))
def test_replay(eng, pkg, golden, name, trivial, erase_p):
    """x and labels_out bit for bit against the replay; pads, rows past h and TAIL elements past x stay NaN; a rerun gives the same
    bits"""
    spec, first, N, crop, pad, epoch, mean, std, C_out, pitch, rows = CASES[name]
    images, labels = dataset(golden, spec)
    img_d, lab_d = dev(images), dev(labels)
    args = (eng, pkg, img_d, lab_d, first, N, trivial, erase_p, crop, pad, 1, epoch, mean, std, C_out, pitch, rows)
    x, lo = run_case(*args)
    want, wl, i, d = TR.batch(images, first, N, trivial, erase_p, crop_size=crop, pad=pad, flip=1, seed=SEED, epoch=epoch, mean=mean,
                              std=std, C_out=C_out, labels=labels)
    for j in range(N):
        assert np.array_equal(x[j], want[j]), (name, j, TR.OPS[d["op"][j]], d["bin"][j], d["sign"][j], bool(d["erase"][j]))
    assert np.array_equal(lo, wl)
    if erase_p:
        assert 0 < d["erase"].sum() < N
    x2, lo2 = run_case(*args)
    assert np.array_equal(x, x2) and np.array_equal(lo, lo2)


def edge_images(n, H, W, C, seed):
    """uint8 [n][H][W][C] cycling through five kinds: flat, one flat channel, two-valued, sparse peaks on a flat ground, random"""
    rng = np.random.default_rng([seed, n, H, W, C])
    img = rng.integers(0, 256, (n, H, W, C), dtype=np.uint8)
    for k in range(n):
        kind = k % 5
        if kind == 0:
            img[k] = rng.integers(0, 256)
        elif kind == 1:
            img[k, ..., 0] = rng.integers(0, 256)
        elif kind == 2:
            img[k] = np.where(rng.random((H, W, C)) < 0.5, rng.integers(0, 128), rng.integers(128, 256))
        elif kind == 3:
            img[k] = np.where(rng.random((H, W, 1)) < 0.02, 255, 7)
    return img, rng.integers(0, 256, n, dtype=np.uint8)


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("trivial", [TR.NEAREST, TR.BILINEAR])
def test_every_op_at_every_bin(eng, pkg, trivial, C):
    """one batch of 4096 crops draws every op at every bin, each signed op with both signs: bit for bit against the replay, flat, one-flat-channel, two-valued and
    sparse crops included, so AutoContrast's flat channels and Equalize's step = 0 run on the device"""
    images, labels = edge_images(4200, 12, 12, C, trivial)
    x, lo = run_case(eng, pkg, dev(images), dev(labels), 50, 4096, trivial, 0.25, pad=1, epoch=6, C_out=8 if C == 3 else 1)
    want, wl, i, d = TR.batch(images, 50, 4096, trivial, 0.25, pad=1, flip=1, seed=SEED, epoch=6, C_out=8 if C == 3 else 1,
                              labels=labels)
    for j in range(len(x)):
        assert np.array_equal(x[j], want[j]), (j, TR.OPS[d["op"][j]], d["bin"][j], d["sign"][j], bool(d["erase"][j]))
    assert np.array_equal(lo, wl)
    pairs = set(zip(d["op"].tolist(), d["bin"].tolist()))
    binned = [k for k, name in enumerate(TR.OPS) if name not in ("Identity", "AutoContrast", "Equalize")]
    assert all((k, b) in pairs for k in binned for b in range(31))
    assert all(set(d["sign"][d["op"] == k].tolist()) == {0, 1} for k, name in enumerate(TR.OPS) if name in TR.SIGNED)
    kinds = i % 5
    for name in ("AutoContrast", "Equalize"):
        assert ((d["op"] == TR.OPS.index(name)) & (kinds == 0)).sum() >= 10               # flat: min = max, step = 0
        assert ((d["op"] == TR.OPS.index(name)) & (kinds == 3)).sum() >= 10               # one dominant byte: step = 0 on most


def test_erase_only_and_none(eng, pkg):
    """trivial NONE with erasing is the plain batch with the boxes zeroed; NONE without erasing is the plain batch"""
    images, labels = synthetic(256, 32, 32, 3)
    for p in (0.0, 1.0):
        x, _ = run_case(eng, pkg, dev(images), dev(labels), 64, 128, TR.NONE, p, pad=4, epoch=7, mean=CIFAR[0], std=CIFAR[1], C_out=8)
        want, _, _, d = TR.batch(images, 64, 128, TR.NONE, p, pad=4, flip=1, seed=SEED, epoch=7, mean=CIFAR[0], std=CIFAR[1], C_out=8)
        assert np.array_equal(x, want)
        plain = A.batch(images, 64, 128, 1, 4, 1, SEED, 7, *CIFAR, 8)[0]
        assert np.array_equal(x, plain) == (p == 0.0)


@pytest.mark.parametrize("trivial", [TR.NEAREST, TR.BILINEAR])
def test_torchvision_on_the_devices_draws(eng, pkg, trivial):
    """torchvision's _apply_op, Normalize and the bf16 cast on the device's own crops and draws: equal on every exact op, and
    differing elsewhere on at most 2 10^-4 of the elements (the CPU test's 200 per 10^6), each bilinear or Sharpness difference by
    one byte step and each NEAREST difference to a neighbouring source pixel"""
    images, labels = synthetic(512, 64, 64, 3)
    N, first = 256, 128
    x, _ = run_case(eng, pkg, dev(images), dev(labels), first, N, trivial, 0.0, crop_size=(56, 56), epoch=4, C_out=3)
    u, i = TR.crops(images, first, N, 1, 0, 1, SEED, 4, (56, 56))
    op, b, sign, _ = TR.draws(i.astype(np.uint64), SEED, 4)
    mags = TR.magnitudes()
    tab = TR.table(56, 56)
    mode = InterpolationMode.NEAREST if trivial == TR.NEAREST else InterpolationMode.BILINEAR
    got = TR.bytes_of(x)
    differ = 0
    for j in range(N):
        t = torch.from_numpy(np.ascontiguousarray(u[j])).permute(2, 0, 1).contiguous()
        want = aa._apply_op(t, TR.OPS[op[j]], TR.magnitude(mags, op[j], b[j], sign[j]), interpolation=mode, fill=None)
        want = want.permute(1, 2, 0).numpy().astype(np.int64)
        d = np.abs(got[j].astype(np.int64) - want)
        if TR.OPS[op[j]] in ("Identity", "Brightness", "Color", "Contrast", "Posterize", "Solarize", "AutoContrast", "Equalize"):
            assert d.max() == 0, (j, TR.OPS[op[j]])
        differ += int((d != 0).sum())
        if trivial == TR.BILINEAR or TR.OPS[op[j]] == "Sharpness":
            assert d.max() <= 1, (j, TR.OPS[op[j]])
        elif d.any():                                   # a NEAREST difference takes a neighbouring source pixel (or the fill)
            ix, iy = TR.grid_coords(56, 56, tab[op[j], b[j], sign[j]])
            nb = neighbours(u[j], ix, iy).astype(np.int64)
            assert np.all(np.any(np.all(nb == want[:, :, None, :], -1), -1)[np.any(d != 0, -1)]), (j, TR.OPS[op[j]])
    print(f"{differ} of {got.size} elements differ from torchvision")
    assert differ <= 2e-4 * got.size


def test_batch_size_does_not_change_the_epoch(eng, pkg):
    """the first 128 positions of an epoch in two batches of 64 equal them in one batch of 128"""
    images, labels = synthetic(512, 32, 32, 3)
    img, lab = dev(images), dev(labels)
    one, l1 = run_case(eng, pkg, img, lab, 0, 128, TR.BILINEAR, 0.5, pad=4, epoch=11, C_out=8)
    a, la = run_case(eng, pkg, img, lab, 0, 64, TR.BILINEAR, 0.5, pad=4, epoch=11, C_out=8)
    b, lb = run_case(eng, pkg, img, lab, 64, 64, TR.BILINEAR, 0.5, pad=4, epoch=11, C_out=8)
    assert np.array_equal(one, np.concatenate([a, b])) and np.array_equal(l1, np.concatenate([la, lb]))


def test_refusals(eng, pkg):
    images, labels = synthetic(64, 8, 8, 3)
    img, lab = dev(images), dev(labels)
    info = pkg.augment_trivial_info(64, 8, 8, 3, 0, 8, pad=2, flip=1, C_out=8)[0]
    x = x_buffer(8, 8, 64)
    ws = torch.zeros(info["ws_bytes"] + 64, dtype=torch.uint8, device=DEV)
    lo = torch.zeros(64, dtype=torch.uint8, device=DEV)
    call = lambda **k: eng.augment_trivial(**dict(dict(images=img, labels=lab, n=64, H=8, W=8, C=3, first=0, N=8, x=x, workspace=ws,
                                                       labels_out=lo, pad=2, flip=1, C_out=8), **k))
    F = "pcnn_augment_trivial_u8_bf16: "
    cases = [
        (dict(images=None), F + "NULL context, images, x or workspace"),
        (dict(workspace=None), "NULL context, images, x or workspace"),
        (dict(labels_out=None), "labels and labels_out must both be NULL or neither"),
        (dict(trivial=5), "trivial = 5: 0 \\(none\\), 1 \\(NEAREST\\) or 2 \\(BILINEAR\\) is required"),
        (dict(erase_p=2.0), "erase_p = 2: a finite 0 <= p <= 1 is required"),
        (dict(crop_size=(6, 6)), "pad = 2: a resized batch takes no padding"),
        (dict(C_out=2), "C_out = 2: C = 3 <= C_out <= 8 is required"),
        (dict(workspace=ws[1:]), "x and the workspace must be 16-byte aligned"),
        (dict(workspace=ws[:info["ws_bytes"] - 16]), f"workspace_bytes = {info['ws_bytes'] - 16}: at least {info['ws_bytes']}"),
        (dict(workspace=x.view(torch.uint8)[:info["ws_bytes"]]), "x must share no byte with images, labels_out or the workspace"),
        (dict(labels_out=ws[:8]), "labels_out must share no byte with labels, images or the workspace"),
        (dict(workspace=img.view(-1)[:info["ws_bytes"]]), "the workspace must share no byte with images or labels"),
    ]
    for change, msg in cases:
        with pytest.raises(pkg.PcnnError, match=msg):
            call(**change)


def test_batcher(eng, pkg, golden):
    """ImageBatcher with trivial_augment and random_erase gives the replay's training batches and the plain eval batches; with the
    defaults it is the plain batcher"""
    images, labels = golden["train_u8"][:512].reshape(-1, 28, 28), golden["train_labels"][:512]
    kw = dict(pad=2, flip=False, seed=SEED, C_out=1, row_pitch=32, image_rows=28)
    b = pkg.ImageBatcher(eng, images, labels, 128, trivial_augment="bilinear", random_erase=0.25, **kw)
    p = pkg.ImageBatcher(eng, images, labels, 128, **kw)
    try:
        b.epoch = p.epoch = 2
        for s in (0, 3):
            ptr, lab = b.batch(s)
            eng.sync()
            x = b.x.to_host().view(np.uint16)[:, :, :28]
            want, wl, _, _ = TR.batch(images[..., None], s * 128, 128, TR.BILINEAR, 0.25, pad=2, flip=0, seed=SEED, epoch=2, labels=labels)
            assert np.array_equal(x, want[..., 0]) and np.array_equal(lab.to_host(), wl)
        b.batch(1, training=False)
        p.batch(1, training=False)
        eng.sync()
        assert np.array_equal(b.x.to_host(), p.x.to_host())
        p.batch(2)
        eng.sync()
        assert np.array_equal(p.x.to_host().view(np.uint16)[:, :, :28],
                              A.batch(images[..., None], 256, 128, 1, 2, 0, SEED, 2, C_out=1)[0][..., 0])
    finally:
        b.close()
        p.close()


def test_resized_batcher(eng, pkg):
    """ImageBatcher with crop_size, trivial_augment and random_erase: the workspace is sized for the crop, training batches are the
    replay's RandomResizedCrop + TrivialAugmentWide + RandomErasing batches into pitched rows, eval batches the resized batcher's"""
    images, labels = synthetic(96, 40, 48, 3)
    kw = dict(flip=True, seed=SEED, mean=IMAGENET[0], std=IMAGENET[1], C_out=8, row_pitch=264, image_rows=34, crop_size=32,
              scale=(0.3, 1.0))
    b = pkg.ImageBatcher(eng, images, labels, 32, trivial_augment="nearest", random_erase=0.5, **kw)
    r = pkg.ImageBatcher(eng, images, labels, 32, **kw)
    try:
        assert b.ws_info["h"] == b.ws_info["w"] == 32 and b.workspace.nbytes == 32 * 32 * 96 * 2
        b.epoch = 1
        for s in (0, 2):
            _, lab = b.batch(s)
            eng.sync()
            x = b.x.to_host().view(np.uint16)
            want, wl, _, _ = TR.batch(images, s * 32, 32, TR.NEAREST, 0.5, crop_size=(32, 32), scale=(0.3, 1.0), flip=1, seed=SEED,
                                      epoch=1, mean=IMAGENET[0], std=IMAGENET[1], C_out=8, labels=labels)
            assert np.array_equal(x[:, :32, :256].reshape(32, 32, 32, 8), want) and np.array_equal(lab.to_host(), wl)
            assert (x[:, 32:] == 0).all() and (x[:, :, 256:] == 0).all()          # the batcher's zeroed pads stay 0
        b.batch(1, training=False)
        r.batch(1, training=False)
        eng.sync()
        assert np.array_equal(b.x.to_host(), r.x.to_host())
    finally:
        b.close()
        r.close()


NB, EPOCHS = ResNetGAP.NB, ResNetGAP.EPOCHS
ERASE = 0.25
ACC_MIN = 0.65            # float32 torch replica 0.7188 (scripts/resnetgap_replica.py --trivial): DESIGN §3.26


def test_resnet_gap_trivial_augmented(eng, pkg, golden):
    """The GAP ResNet trained on batches with a shuffle, a pad-2 crop, TrivialAugmentWide (BILINEAR) and RandomErasing(ERASE): the
    first 5 batches and labels are bit-exact against the replay, a fresh run reproduces the parameters after 5 steps, the loss
    falls, and test accuracy, evaluated through the batcher's plain eval path, exceeds ACC_MIN"""
    train_u8 = golden["train_u8"].reshape(-1, 28, 28)
    aug = pkg.ImageBatcher(eng, train_u8, golden["train_labels"], NB, pad=2, shuffle=True, seed=SEED, row_pitch=32, image_rows=28,
                           trivial_augment="bilinear", random_erase=ERASE)
    tests = pkg.ImageBatcher(eng, golden["test_u8"].reshape(-1, 28, 28), golden["test_labels"], NB, row_pitch=32, image_rows=28)
    make = lambda: ResNetGAP(eng, pkg, ResNetGAP.init_params())
    tab = TR.table(28, 28)

    def replayed(net, step, x, lab):
        xb = aug.x.to_host()
        wx, wl, *_ = TR.batch(train_u8[..., None], step * NB, NB, TR.BILINEAR, ERASE, pad=2, seed=SEED, epoch=0,
                              labels=golden["train_labels"], tab=tab)
        assert np.array_equal(xb[:, :, :28], wx.reshape(NB, 28, 28)) and (xb[:, :, 28:] == 0).all()
        assert np.array_equal(lab.to_host(), wl)
        net.forward(x, lab)
        net.backward()

    try:
        loss, acc, _ = train(eng, pkg, golden, make, EPOCHS, batches=aug, tests=tests, check_step=replayed)
    finally:
        aug.close()
        tests.close()
    print(f"GAP ResNet on TrivialAugmentWide + RandomErasing({ERASE}): mean loss {loss[0]:.4f} -> {loss[-1]:.4f}, test accuracy "
          f"{acc:.4f} (threshold {ACC_MIN})")
    assert np.isfinite(loss).all() and loss[-1] < loss[0]
    assert acc > ACC_MIN
