"""The input pipeline on the device (pcnn_augment_u8_bf16, ImageBatcher): x and labels_out bit for bit against the numpy replay of
augment_ref.py in the example networks' MNIST layout, CIFAR-sized RGB into the row-Toeplitz (C_out 3) and wide (C_out 8) layouts,
odd shapes with pitched rows and padded images, pad > H, N = 1, N = n, batches in mid-epoch and an ImageNet-sized batch from a
dataset larger than L2; untouched pads and tails, reruns, batch sizes that split an epoch differently, every image once per
epoch, the eval path against mnist_device, torch eager building the same batch, refusals; and the GAP ResNet of
example_nets trained through the batcher, first as a drop-in for its pre-converted slices, then with a shuffle and a
random crop."""
import numpy as np
import pytest
import torch

import augment_ref as A
from augment_ref import torch_batch
from example_nets import DEV, NAN_BF16, ResNetGAP, Slices, mnist_device, same_bits, train

pytestmark = pytest.mark.gpu

NB, EPOCHS, LR_STEP = ResNetGAP.NB, ResNetGAP.EPOCHS, ResNetGAP.LR_STEP
ACC_MIN = 0.88            # the threshold of the GAP ResNet trained on the pre-converted slices (test_avgpool_nhwc_gpu)
TAIL = 64                 # elements past x that must stay untouched
LABEL_SENTINEL = 0xAA
SEED = 0x0123456789ABCDEF
CIFAR = ((0.4914, 0.4822, 0.4465), (0.2470, 0.2435, 0.2616))
IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))


def synthetic(n, H, W, C, seed=0):
    """uint8 [n][H][W][C] holding every byte value (the first 256 bytes of each image are 0 .. 255 rotated by the index), random
    elsewhere, and labels [n]"""
    rng = np.random.default_rng([seed, n, H, W, C])
    img = rng.integers(0, 256, (n, H * W * C), dtype=np.uint8)
    k = min(256, H * W * C)
    img[:, :k] = (np.arange(k)[None, :] + np.arange(n)[:, None]) % 256
    return img.reshape(n, H, W, C), rng.integers(0, 256, n, dtype=np.uint8)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def x_buffer(N, rows, pitch):
    """a flat int16 buffer of N rows pitch + TAIL elements, every one NaN"""
    return torch.full((N * rows * pitch + TAIL,), NAN_BF16, dtype=torch.int16, device=DEV)


def bits(t):
    return t.cpu().numpy().view(np.uint16)


def run_case(eng, pkg, images, labels, first, N, shuffle, pad, flip, epoch, mean=None, std=None, C_out=None, row_pitch=0, image_rows=0):
    """one call on fresh NaN-filled buffers: (x [N][image_rows][pitch] bits, labels_out, info) after checking pads and tails"""
    n, H, W, C = images.shape
    C_out = C if C_out is None else C_out
    info, _ = pkg.augment_info(n, H, W, C, first, N, shuffle, pad, flip, C_out, row_pitch, image_rows, mean, std)
    rows, pitch = info["image_rows"], info["row_pitch"]
    img_d = images if torch.is_tensor(images) else dev(images)
    lab_d = None if labels is None else (labels if torch.is_tensor(labels) else dev(labels))
    x = x_buffer(N, rows, pitch)
    lo = None if labels is None else torch.full((N + TAIL,), LABEL_SENTINEL, dtype=torch.uint8, device=DEV)
    eng.augment(img_d, lab_d, n, H, W, C, first, N, x, lo, shuffle=shuffle, pad=pad, flip=flip, seed=SEED, epoch=epoch, mean=mean,
                std=std, C_out=C_out, row_pitch=row_pitch, image_rows=image_rows)
    xb = bits(x)
    assert (xb[N * rows * pitch:] == NAN_BF16).all()                      # past x
    xb = xb[:N * rows * pitch].reshape(N, rows, pitch)
    assert (xb[:, :, W * C_out:] == NAN_BF16).all() and (xb[:, H:, :] == NAN_BF16).all()     # pad columns and pad rows
    lob = None
    if lo is not None:
        lob = lo.cpu().numpy()
        assert (lob[N:] == LABEL_SENTINEL).all()
        lob = lob[:N]
    return xb, lob, info


def want(images, labels, first, N, shuffle, pad, flip, epoch, mean=None, std=None, C_out=None):
    images = images.cpu().numpy() if torch.is_tensor(images) else images
    labels = labels.cpu().numpy() if torch.is_tensor(labels) else labels
    return A.batch(images, first, N, shuffle, pad, flip, SEED, epoch, mean, std, C_out, labels)


CASES = {  # name: (dataset (n, H, W, C) or "mnist", first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows)
    "mnist-28x28-rows32": ("mnist", 128, 128, 1, 2, 0, 3, None, None, 1, 32, 28),
    "cifar-32x32x3-cout3": ((2048, 32, 32, 3), 512, 256, 1, 4, 1, 1, *CIFAR, 3, 0, 0),
    "cifar-32x32x3-cout8": ((2048, 32, 32, 3), 512, 256, 1, 4, 1, 1, *CIFAR, 8, 0, 0),
    "odd-27x31x1-pitched": ((100, 27, 31, 1), 3, 7, 1, 3, 1, 5, (0.3,), (0.7,), 1, 40, 30),
    "odd-5x7x4-cout5": ((50, 5, 7, 4), 11, 9, 1, 2, 1, 2, (-0.5, 0.0, 0.25, 1.0), (1e-3, 2.0, 0.5, 1.0), 5, 48, 8),
    "pad-over-H": ((64, 6, 6, 2), 0, 16, 1, 9, 1, 7, None, None, 8, 0, 0),
    "N1-last": ((10, 8, 8, 3), 9, 1, 1, 4, 1, 0, *IMAGENET, 8, 0, 0),
    "N-equals-n": ((300, 12, 12, 1), 0, 300, 1, 1, 1, 1 << 40, None, None, 1, 16, 0),
    "no-shuffle-cifar": ((256, 32, 32, 3), 64, 64, 0, 4, 1, 2, *CIFAR, 8, 0, 0),
    "imagenet-224-cout8": ((512, 224, 224, 3), 256, 256, 1, 4, 1, 1, *IMAGENET, 8, 0, 0),
}


def dataset(golden, spec):
    if spec == "mnist":
        return golden["train_u8"].reshape(-1, 28, 28, 1), golden["train_labels"]
    return synthetic(*spec)


@pytest.mark.parametrize("name", list(CASES))
def test_replay(eng, pkg, golden, name):
    """x and labels_out bit for bit against the replay; pads, rows past H and TAIL elements past x stay NaN; a rerun gives the
    same bits"""
    spec, first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows = CASES[name]
    images, labels = dataset(golden, spec)
    img_d, lab_d = dev(images), dev(labels)
    xb, lob, info = run_case(eng, pkg, img_d, lab_d, first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows)
    H, W = images.shape[1:3]
    wx, wl, i, oy, ox, fl = want(images, labels, first, N, shuffle, pad, flip, epoch, mean, std, C_out)
    got = xb[:, :H, :W * C_out].reshape(wx.shape)
    assert np.array_equal(got, wx), np.argwhere(got != wx)[:5]
    assert np.array_equal(lob, wl)
    if pad and N > 1:
        assert len(set(zip(oy.tolist(), ox.tolist()))) > 1           # the crops move
    xb2, lob2, _ = run_case(eng, pkg, img_d, lab_d, first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows)
    assert np.array_equal(xb, xb2) and np.array_equal(lob, lob2)
    print(f"{name}: vec {info['vec']}, grid {info['grid']}, rows per CTA {info['rows_per_cta']}, b {info['b']}")


@pytest.mark.parametrize("name", ["cifar-32x32x3-cout8", "odd-5x7x4-cout5", "imagenet-224-cout8"])
def test_torch_eager_builds_the_same_batch(eng, pkg, golden, name):
    spec, first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows = CASES[name]
    images, labels = dataset(golden, spec)
    img_d = dev(images)
    xb, _, _ = run_case(eng, pkg, img_d, dev(labels), first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows)
    _, _, i, oy, ox, fl = want(images, None, first, N, shuffle, pad, flip, epoch, mean, std, C_out)
    H, W = images.shape[1:3]
    tb = torch_batch(img_d, i, oy, ox, fl, pad, mean, std, C_out).view(torch.int16).cpu().numpy().view(np.uint16)
    assert np.array_equal(xb[:, :H, :W * C_out].reshape(tb.shape), tb)


def test_batch_size_does_not_change_the_epoch(eng, pkg):
    """an epoch's batches at N = 64, concatenated, equal its batches at N = 128, x and labels"""
    images, labels = synthetic(1024, 32, 32, 3)
    img_d, lab_d = dev(images), dev(labels)
    out = {}
    for N in (64, 128):
        b = pkg.ImageBatcher(eng, img_d, lab_d, N, pad=4, flip=True, shuffle=True, seed=SEED, mean=CIFAR[0], std=CIFAR[1], C_out=8)
        b.epoch = 6
        xs, ls = [], []
        for s in range(b.steps_per_epoch):
            b.batch(s)
            xs.append(b.x.to_host())
            ls.append(b.labels_out.to_host())
        out[N] = np.concatenate(xs), np.concatenate(ls)
        b.close()
    assert np.array_equal(out[64][0], out[128][0]) and np.array_equal(out[64][1], out[128][1])


def test_every_image_once_per_epoch(eng, pkg):
    """the dataset index, written into pixel (0, 0) of each image, comes back exactly once per epoch; n = 1000 is not a multiple
    of N = 128, so the last 104 positions of the epoch are dropped and the batches cover the first 896"""
    n = 1000
    images = np.zeros((n, 8, 8, 2), np.uint8)
    images[:, 0, 0, 0], images[:, 0, 0, 1] = np.arange(n) & 255, np.arange(n) >> 8
    for N, covered in ((100, n), (128, 896)):
        b = pkg.ImageBatcher(eng, images, None, N, shuffle=True, seed=SEED)
        assert b.steps_per_epoch == n // N and b.labels_out is None
        for epoch in (0, 1):
            b.epoch = epoch
            seen = []
            for s in range(b.steps_per_epoch):
                x, lab = b.batch(s)
                assert x == b.x.ptr and lab is None
                u = np.rint(pkg.bf16_bits_to_f32(b.x.to_host()[:, 0, :2]) * 255).astype(np.int64)
                seen.append(u[:, 0] + 256 * u[:, 1])
            seen = np.concatenate(seen)
            assert np.array_equal(seen, A.indices(n, 0, covered, 1, SEED, epoch))
            if covered == n:
                assert np.array_equal(np.sort(seen), np.arange(n))
        b.close()


def test_eval_path_is_mnist_device(eng, pkg, golden):
    """training=False (identity order, no crop, no flip) with mean 0 / std 1 gives exactly the bits of mnist_device, pad columns
    included (the batcher's x starts zeroed and the pad is never written)"""
    b = pkg.ImageBatcher(eng, golden["test_u8"].reshape(-1, 28, 28), golden["test_labels"], NB, pad=2, flip=True, shuffle=True,
                         seed=SEED, row_pitch=32, image_rows=28)
    old = bits(mnist_device(pkg, golden["test_u8"])).reshape(-1, NB, 28, 32)
    for s in range(b.steps_per_epoch):
        _, lab = b.batch(s, training=False)
        assert np.array_equal(b.x.to_host(), old[s])
        assert np.array_equal(lab.to_host(), golden["test_labels"][s * NB:(s + 1) * NB])
    with pytest.raises(pkg.PcnnError, match="step = 2: 0 <= step < steps_per_epoch = 2"):
        b.batch(2)
    b.close()


def test_refusals(eng, pkg):
    images, labels = synthetic(64, 8, 8, 3)
    img, lab = dev(images), dev(labels)
    x = x_buffer(8, 8, 64)
    lo = torch.zeros(64, dtype=torch.uint8, device=DEV)
    call = lambda **k: eng.augment(**dict(dict(images=img, labels=lab, n=64, H=8, W=8, C=3, first=0, N=8, x=x, labels_out=lo, shuffle=1,
                                               pad=2, flip=1, C_out=8), **k))
    cases = [
        (dict(images=None), "pcnn_augment_u8_bf16: NULL context, images or x"),
        (dict(x=None), "NULL context, images or x"),
        (dict(labels_out=None), "labels and labels_out must both be NULL or neither"),
        (dict(labels=None), "labels and labels_out must both be NULL or neither"),
        (dict(x=x.data_ptr() + 2), "x must be 16-byte aligned"),
        (dict(x=img), "overlapping buffers: x must share no byte with images or labels_out"),
        (dict(labels_out=x.data_ptr() + 64), "overlapping buffers: x must share no byte"),
        (dict(labels_out=lab.data_ptr() + 8), "overlapping buffers: labels_out must share no byte with labels or images"),
        (dict(labels_out=img.data_ptr() + 100), "labels_out must share no byte"),
        (dict(first=57), "pcnn_augment_u8_bf16: first = 57, N = 8: 0 <= first"),
        (dict(C_out=2), "pcnn_augment_u8_bf16: C_out = 2"),
        (dict(pad=65), "pcnn_augment_u8_bf16: pad = 65"),
        (dict(shuffle=2), "shuffle = 2, flip = 1: each must be 0 or 1"),
        (dict(std=(1.0, 0.0, 1.0)), "std\\[1\\] = 0: a finite std > 0 is required"),
        (dict(row_pitch=12), "row_pitch = 12"),
    ]
    for change, msg in cases:
        with pytest.raises(pkg.PcnnError, match=msg):
            call(**change)
    call()
    eng.sync()
    assert (bits(x)[8 * 8 * 64:] == NAN_BF16).all()
    img_odd = torch.zeros(64 * 192 + 1, dtype=torch.uint8, device=DEV)[1:]       # an unaligned dataset base is accepted
    img_odd.copy_(img.reshape(-1))
    xb, _, _ = run_case(eng, pkg, img_odd.reshape(64, 8, 8, 3), lab, 0, 8, 1, 2, 1, 0, C_out=8)
    assert np.array_equal(xb[:, :8, :64].reshape(8, 8, 8, 8), want(images, labels, 0, 8, 1, 2, 1, 0, C_out=8)[0])


# ------------------------------------------------------------------------------------------------ end to end
def mnist_batcher(pkg, eng, golden, **k):
    return pkg.ImageBatcher(eng, golden["train_u8"].reshape(-1, 28, 28), golden["train_labels"], NB, row_pitch=32, image_rows=28, **k)


def test_resnet_gap_through_the_batcher(eng, pkg, golden):
    """(a) Drop-in: shuffle 0, pad 0, flip 0, mean 0 / std 1 gives every batch of mnist_device's slices, and the parameters after 5
    SGD steps equal, bit for bit, those of a run fed the slices.  (b) Augmented: shuffle, pad 2, no flip (digits are not mirror
    images): the first 5 batches and labels are bit-exact against the replay, a fresh run reproduces the parameters after 5
    steps, the loss falls over EPOCHS epochs and test accuracy, evaluated through the batcher with training=False, exceeds
    ACC_MIN."""
    slices = Slices(pkg, golden["train_u8"], golden["train_labels"], NB)
    net = ResNetGAP(eng, pkg, ResNetGAP.init_params())
    try:
        for s in range(5):
            net.forward(*slices.batch(s))
            net.backward()
            net.sgd(LR_STEP)
        eng.sync()
        old5 = net.params()
    finally:
        net.close()

    make = lambda: ResNetGAP(eng, pkg, ResNetGAP.init_params())
    tests = pkg.ImageBatcher(eng, golden["test_u8"].reshape(-1, 28, 28), golden["test_labels"], NB, row_pitch=32, image_rows=28)
    plain = mnist_batcher(pkg, eng, golden, shuffle=False)
    old = bits(slices.x).reshape(-1, NB, 28, 32)

    def same_as_slices(net, step, x, lab):
        assert np.array_equal(plain.x.to_host(), old[step]) and np.array_equal(lab.to_host(), golden["train_labels"][step * NB:(step + 1) * NB])
        net.forward(x, lab)
        net.backward()

    loss_plain, acc_plain, p5 = train(eng, pkg, golden, make, EPOCHS, batches=plain, tests=tests, check_step=same_as_slices)
    plain.close()
    assert same_bits(p5, old5)

    train_u8 = golden["train_u8"].reshape(-1, 28, 28, 1)
    aug = mnist_batcher(pkg, eng, golden, pad=2, flip=False, shuffle=True, seed=SEED)

    def replayed(net, step, x, lab):
        xb = aug.x.to_host()
        wx, wl, *_ = A.batch(train_u8, step * NB, NB, 1, 2, 0, SEED, 0, labels=golden["train_labels"])
        assert np.array_equal(xb[:, :, :28], wx.reshape(NB, 28, 28)) and (xb[:, :, 28:] == 0).all()
        assert np.array_equal(lab.to_host(), wl)
        net.forward(x, lab)
        net.backward()

    loss_aug, acc_aug, _ = train(eng, pkg, golden, make, EPOCHS, batches=aug, tests=tests, check_step=replayed)
    aug.close()
    tests.close()
    print(f"GAP ResNet through the batcher: plain mean loss {loss_plain[0]:.4f} -> {loss_plain[-1]:.4f}, test accuracy {acc_plain:.4f}; "
          f"shuffle + crop (pad 2) {loss_aug[0]:.4f} -> {loss_aug[-1]:.4f}, test accuracy {acc_aug:.4f} (threshold {ACC_MIN})")
    assert np.isfinite(loss_aug).all() and loss_aug[-1] < loss_aug[0]
    assert acc_plain > ACC_MIN and acc_aug > ACC_MIN
