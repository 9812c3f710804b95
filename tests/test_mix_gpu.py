"""Mixed batches and soft targets on the device (pcnn_augment_mix_u8_bf16, pcnn_softmax_ce_soft_bf16, ImageBatcher's mixup_alpha /
cutmix_alpha): x, labels_out and labels_b_out bit for bit against mix_ref's replay for MixUp and CutMix over the shapes of
test_augment_gpu, torchvision's v2.MixUp / v2.CutMix building the same batch from torch's fp32 eager batch, the edge cases that
reduce to the plain batch, untouched pads and tails, reruns and refusals; the soft loss against its float64 replay and, at lam = 1
with eps = 0, against pcnn_softmax_ce_bf16 bit for bit; and the GAP ResNet of example_nets trained on mixed batches with label
smoothing."""
from unittest import mock

import numpy as np
import pytest
import torch
from torchvision.transforms import v2

import augment_ref as A
import linear_ref as LR
import mix_ref as M
from example_nets import DEV, NAN_BF16, ResNetGAP, nan_buf, same_bits, train
from test_augment_gpu import CASES, LABEL_SENTINEL, SEED, TAIL, bits, dataset, dev, x_buffer

pytestmark = pytest.mark.gpu

NB, EPOCHS, LR_STEP = ResNetGAP.NB, ResNetGAP.EPOCHS, ResNetGAP.LR_STEP
ALPHAS, EPS = (0.2, 1.0), 0.1       # mixup_alpha, cutmix_alpha and label smoothing of the end-to-end run (scripts/replica.py)
ACC_MIN = 0.80                      # scripts/resnetgap_replica.py --mix 0.2 reaches 0.8633 (DESIGN 3.24)


def box_for(H, W):
    """a box that cuts across both dimensions without covering either"""
    return (W // 4, H // 3, max(W // 4 + 1, W - W // 5), max(H // 3 + 1, H - 1))


def run_mix(eng, pkg, images, labels, first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows, mode, lam, box):
    """one mixed call on fresh NaN-filled buffers: (x [N][image_rows][pitch] bits, labels_out, labels_b_out) after checking pads
    and tails"""
    n, H, W, C = images.shape
    info, _ = pkg.augment_info(n, H, W, C, first, N, shuffle, pad, flip, C_out, row_pitch, image_rows, mean, std)
    rows, pitch = info["image_rows"], info["row_pitch"]
    x = x_buffer(N, rows, pitch)
    lo = torch.full((N + TAIL,), LABEL_SENTINEL, dtype=torch.uint8, device=DEV)
    lb = torch.full((N + TAIL,), LABEL_SENTINEL, dtype=torch.uint8, device=DEV)
    eng.augment_mix(images, labels, n, H, W, C, first, N, x, lo, lb, mode=mode, lam=lam, box=box, shuffle=shuffle, pad=pad, flip=flip,
                    seed=SEED, epoch=epoch, mean=mean, std=std, C_out=C_out, row_pitch=row_pitch, image_rows=image_rows)
    xb = bits(x)
    assert (xb[N * rows * pitch:] == NAN_BF16).all()                                        # past x
    xb = xb[:N * rows * pitch].reshape(N, rows, pitch)
    assert (xb[:, :, W * C_out:] == NAN_BF16).all() and (xb[:, H:, :] == NAN_BF16).all()     # pad columns and pad rows
    lo, lb = lo.cpu().numpy(), lb.cpu().numpy()
    assert (lo[N:] == LABEL_SENTINEL).all() and (lb[N:] == LABEL_SENTINEL).all()
    return xb, lo[:N], lb[:N]


def plain_call(eng, pkg, images, labels, first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows):
    n, H, W, C = images.shape
    info, _ = pkg.augment_info(n, H, W, C, first, N, shuffle, pad, flip, C_out, row_pitch, image_rows, mean, std)
    x = x_buffer(N, info["image_rows"], info["row_pitch"])
    lo = torch.zeros(N, dtype=torch.uint8, device=DEV)
    eng.augment(images, labels, n, H, W, C, first, N, x, lo, shuffle=shuffle, pad=pad, flip=flip, seed=SEED, epoch=epoch, mean=mean,
                std=std, C_out=C_out, row_pitch=row_pitch, image_rows=image_rows)
    return bits(x)[:N * info["image_rows"] * info["row_pitch"]].reshape(N, info["image_rows"], info["row_pitch"])


MODES = {"mixup": (M.MIXUP, 0.37), "cutmix": (M.CUTMIX, None)}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", [c for c in CASES if c != "imagenet-224-cout8"] + ["N1-only"])
def test_replay(eng, pkg, golden, name, mode):
    """x, labels_out and labels_b_out bit for bit against the replay; pads, rows past H and TAIL elements past x stay NaN, the
    label tails their sentinel; a rerun gives the same bits"""
    if name == "N1-only":                                       # N = 1 = n: the partner is the image itself
        spec, first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows = ((1, 9, 11, 2), 0, 1, 1, 3, 1, 4, None,
                                                                                              None, 2, 0, 0)
    else:
        spec, first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows = CASES[name]
    images, labels = dataset(golden, spec)
    H, W = images.shape[1:3]
    m, lam = MODES[mode]
    box = box_for(H, W) if m == M.CUTMIX else (0, 0, 0, 0)
    lam = lam if lam is not None else 1.0 - (box[2] - box[0]) * (box[3] - box[1]) / (W * H)
    img_d, lab_d = dev(images), dev(labels)
    args = (img_d, lab_d, first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows, m, lam, box)
    xb, lo, lb = run_mix(eng, pkg, *args)
    wx, wl, wlb = M.batch(images, first, N, m, lam, box, shuffle, pad, flip, SEED, epoch, mean, std, C_out, labels)
    got = xb[:, :H, :W * C_out].reshape(wx.shape)
    assert np.array_equal(got, wx), np.argwhere(got != wx)[:5]
    assert np.array_equal(lo, wl) and np.array_equal(lb, wlb)
    assert np.array_equal(lb, np.roll(wl, 1))
    xb2, lo2, lb2 = run_mix(eng, pkg, *args)
    assert np.array_equal(xb, xb2) and np.array_equal(lo, lo2) and np.array_equal(lb, lb2)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", ["cifar-32x32x3-cout8", "odd-5x7x4-cout5", "mnist-28x28-rows32"])
def test_torchvision_builds_the_same_batch(eng, pkg, golden, name, mode):
    """torch's fp32 eager batch through v2.MixUp / v2.CutMix, make_params returning the call's lam or box, then cast to bf16, has
    the device's bits; the mixed labels equal mix_ref's m"""
    spec, first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows = CASES[name]
    images, labels = dataset(golden, spec)
    n, H, W, C = images.shape
    m, lam = MODES[mode]
    box = box_for(H, W) if m == M.CUTMIX else (0, 0, 0, 0)
    lam = lam if lam is not None else 1.0 - (box[2] - box[0]) * (box[3] - box[1]) / (W * H)
    img_d, lab_d = dev(images), dev(labels)
    xb, lo, lb = run_mix(eng, pkg, img_d, lab_d, first, N, shuffle, pad, flip, epoch, mean, std, C_out, row_pitch, image_rows, m, lam, box)
    _, _, i, oy, ox, fl = A.batch(images, first, N, shuffle, pad, flip, SEED, epoch, mean, std, C_out)
    f32 = M.torch_f32_batch(img_d, i, oy, ox, fl, pad, mean, std)
    tf = v2.MixUp(alpha=1.0, num_classes=256) if m == M.MIXUP else v2.CutMix(alpha=1.0, num_classes=256)
    params = dict(lam=lam) if m == M.MIXUP else dict(box=box, lam_adjusted=lam)
    with mock.patch.object(tf, "make_params", return_value=params):
        out, mixed = tf(f32, torch.from_numpy(labels[i].astype(np.int64)).to(DEV))
    tb = out.permute(0, 2, 3, 1).to(torch.bfloat16).view(torch.int16).cpu().numpy().view(np.uint16)
    got = xb[:, :H, :W * C_out].reshape(N, H, W, C_out)
    assert np.array_equal(got[..., :C], tb) and (got[..., C:] == 0).all()
    want_m, _ = M.soft_target(lo, lb, lam, 0.0, 256)
    assert np.array_equal(mixed.cpu().numpy().view(np.uint32), want_m.view(np.uint32))


def test_edge_cases_reduce_to_the_plain_batch(eng, pkg):
    """MixUp at lam = 1 and CutMix with an empty box give the plain call's batch; a full box gives the plain batch rolled by one"""
    images, labels = dataset(None, (300, 12, 12, 3))
    img_d, lab_d = dev(images), dev(labels)
    common = (img_d, lab_d, 32, 64, 1, 2, 1, 3, (0.2, 0.3, 0.4), (0.5, 0.25, 1.5), 8, 0, 0)
    plain = plain_call(eng, pkg, *common)
    for mode, lam, box in ((M.MIXUP, 1.0, (0, 0, 0, 0)), (M.CUTMIX, 1.0, (0, 0, 0, 0)), (M.CUTMIX, 1.0, (5, 3, 5, 12)),
                           (M.CUTMIX, 0.0, (0, 0, 12, 12))):
        xb, lo, lb = run_mix(eng, pkg, *common, mode, lam, box)
        full = box == (0, 0, 12, 12)
        assert np.array_equal(xb, np.roll(plain, 1, axis=0) if full else plain), (mode, lam, box)
    xb, _, _ = run_mix(eng, pkg, *common, M.MIXUP, 0.0, (0, 0, 0, 0))
    assert np.array_equal(xb, np.roll(plain, 1, axis=0))                  # lam = 0: the partner alone


def test_refusals(eng, pkg):
    images, labels = dataset(None, (64, 8, 8, 3))
    img, lab = dev(images), dev(labels)
    x = x_buffer(8, 8, 64)
    lo = torch.zeros(64, dtype=torch.uint8, device=DEV)
    lb = torch.zeros(64, dtype=torch.uint8, device=DEV)
    call = lambda **k: eng.augment_mix(**dict(dict(images=img, labels=lab, n=64, H=8, W=8, C=3, first=0, N=8, x=x, labels_out=lo,
                                                   labels_b_out=lb, mode=M.CUTMIX, lam=0.5, box=(1, 2, 5, 8), shuffle=1, pad=2, flip=1,
                                                   C_out=8), **k))
    cases = [
        (dict(images=None), "pcnn_augment_mix_u8_bf16: NULL context, images or x"),
        (dict(labels_out=None), "pcnn_augment_mix_u8_bf16: labels and labels_out must both be NULL or neither"),
        (dict(x=x.data_ptr() + 2), "pcnn_augment_mix_u8_bf16: x must be 16-byte aligned"),
        (dict(first=57), "pcnn_augment_mix_u8_bf16: first = 57, N = 8: 0 <= first"),
        (dict(mode=0), "mode = 0: 1 \\(MixUp\\) or 2 \\(CutMix\\) is required"),
        (dict(mode=3), "mode = 3: 1 \\(MixUp\\) or 2 \\(CutMix\\) is required"),
        (dict(lam=-0.25), "lam = -0.25: a finite 0 <= lam <= 1 is required"),
        (dict(lam=1.5), "lam = 1.5: a finite 0 <= lam <= 1 is required"),
        (dict(lam=float("nan")), "lam = nan: a finite 0 <= lam <= 1 is required"),
        (dict(lam=float("inf")), "lam = inf: a finite"),
        (dict(box=(-1, 0, 4, 4)), "x1 = -1, x2 = 4: 0 <= x1 <= x2 <= W = 8 is required"),
        (dict(box=(5, 0, 4, 4)), "x1 = 5, x2 = 4: 0 <= x1 <= x2 <= W = 8"),
        (dict(box=(0, 0, 9, 4)), "x1 = 0, x2 = 9: 0 <= x1 <= x2 <= W = 8"),
        (dict(box=(0, -2, 4, 4)), "y1 = -2, y2 = 4: 0 <= y1 <= y2 <= H = 8 is required"),
        (dict(box=(0, 5, 4, 4)), "y1 = 5, y2 = 4"),
        (dict(box=(0, 0, 4, 9)), "y1 = 0, y2 = 9"),
        (dict(labels_b_out=None), "labels and labels_b_out must both be NULL or neither"),
        (dict(labels=None, labels_out=None), "labels and labels_b_out must both be NULL or neither"),
        (dict(labels_b_out=x.data_ptr() + 64), "overlapping buffers: labels_b_out must share no byte with x, images, labels or labels_out"),
        (dict(labels_b_out=img.data_ptr() + 100), "labels_b_out must share no byte"),
        (dict(labels_b_out=lab.data_ptr() + 8), "labels_b_out must share no byte"),
        (dict(labels_b_out=lo.data_ptr() + 4), "labels_b_out must share no byte"),
    ]
    for change, msg in cases:
        with pytest.raises(pkg.PcnnError, match=msg):
            call(**change)
    call()
    call(labels=None, labels_out=None, labels_b_out=None, mode=M.MIXUP)
    eng.sync()
    assert (bits(x)[8 * 8 * 64:] == NAN_BF16).all()
    with pytest.raises(pkg.PcnnError, match="pcnn_softmax_ce_soft_bf16: lam = 2: a finite 0 <= lam <= 1"):
        eng.softmax_ce_soft_bf16(x, lo, 8, 10, 1.0, nan_buf(8, 10), labels_b=lb, lam=2.0)
    with pytest.raises(pkg.PcnnError, match="lam = nan"):
        eng.softmax_ce_soft_bf16(x, lo, 8, 10, 1.0, nan_buf(8, 10), lam=float("nan"))
    with pytest.raises(pkg.PcnnError, match="smoothing = -0.1: 0 <= smoothing <= 1 is required"):
        eng.softmax_ce_soft_bf16(x, lo, 8, 10, 1.0, nan_buf(8, 10), smoothing=-0.1)
    with pytest.raises(pkg.PcnnError, match="smoothing = nan"):
        eng.softmax_ce_soft_bf16(x, lo, 8, 10, 1.0, nan_buf(8, 10), smoothing=float("nan"))
    with pytest.raises(pkg.PcnnError, match="smoothing = 1.5"):
        eng.softmax_ce_soft_bf16(x, lo, 8, 10, 1.0, nan_buf(8, 10), smoothing=1.5)
    with pytest.raises(pkg.PcnnError, match="pcnn_softmax_ce_soft_bf16: N = 8, O = 257"):
        eng.softmax_ce_soft_bf16(x, lo, 8, 257, 1.0, nan_buf(8, 257))
    with pytest.raises(pkg.PcnnError, match="pcnn_softmax_ce_soft_bf16: NULL context, logits, labels or dlogits"):
        eng.softmax_ce_soft_bf16(x, None, 8, 10, 1.0, nan_buf(8, 10))
    with pytest.raises(pkg.PcnnError, match="pcnn_softmax_ce_soft_bf16: dlogits overlaps logits"):
        eng.softmax_ce_soft_bf16(x, lo, 8, 10, 1.0, x.data_ptr() + 16)


# ------------------------------------------------------------------------------------------------ soft-target loss
def check_soft(pkg, zb, labels, labels_b, lam, eps, scale, dh, lh, ph):
    """dlogits bits against the replay (one bf16 ulp allowed within 1e-12 of a rounding boundary), loss within 1e-6, pred exact;
    returns the count of one-ulp values"""
    g, lref, pref, _ = M.softmax_ce_soft_f64(pkg.bf16_bits_to_f32(zb), labels, labels_b, lam, eps, np.float32(scale))
    nan = np.isnan(g)
    assert np.array_equal(np.isnan(pkg.bf16_bits_to_f32(dh)), nan)
    exp = LR.f64_to_bf16_bits(pkg, np.where(nan, 0, g))
    diff = np.abs(dh.astype(np.int64) - exp.astype(np.int64))
    near = LR.near_boundary(pkg, np.where(nan, 0, g)) & ~nan
    assert np.all((diff[~nan] == 0) | (near[~nan] & (diff[~nan] <= 1)))
    if lh is not None:
        assert np.array_equal(np.isnan(lh), np.isnan(lref))
        ok = ~np.isnan(lref)
        assert np.all(np.abs(lh[ok] - lref[ok]) <= 1e-6 * np.maximum(1.0, np.abs(lref[ok])))
    if ph is not None:
        assert np.array_equal(ph, pref)
    return int((diff[~nan] != 0).sum())


@pytest.mark.parametrize("O", [1, 10, 37, 256])
def test_softmax_ce_soft_bf16(eng, pkg, O):
    """for lam in {0, 0.3, 1} and eps in {0, 0.1, 1}, with and without labels_b: dlogits, loss and pred against the replay with
    ties, NaN rows, -Inf rows and labels or label_b >= O; in place gives the same bits"""
    N = 515
    rng = np.random.default_rng(O + 1000)
    z = np.where(rng.random((N, O)) < 0.5, rng.integers(-4, 5, (N, O)) / 2.0, rng.normal(0, 3, (N, O))).astype(np.float32)
    z[::7] = rng.integers(-2, 3, (len(z[::7]), O)) / 2.0
    z[5, O // 2] = np.nan
    z[11] = -np.inf
    zb = pkg.f32_to_bf16_bits(z)
    labels = rng.integers(0, O, N).astype(np.uint8)
    labels_b = rng.integers(0, O, N).astype(np.uint8)
    labels[[3, 17]] = [O, 255] if O < 255 else [255, 255]
    labels_b[[4, 18]] = [O, 255] if O < 255 else [255, 255]
    labels_b[20:40] = labels[20:40]
    zd = torch.from_numpy(zb.view(np.int16)).to(DEV)
    lab, labb = torch.from_numpy(labels).to(DEV), torch.from_numpy(labels_b).to(DEV)
    scale = 1.0 / N
    ulps = 0
    for lam in (0.0, 0.3, 1.0):
        for eps in (0.0, 0.1, 1.0):
            for lb_h, lb_d in ((labels_b, labb), (None, None)):
                d = nan_buf(N, O)
                loss = torch.full((N,), float("nan"), dtype=torch.float32, device=DEV)
                pred = torch.full((N,), -7, dtype=torch.int32, device=DEV)
                eng.softmax_ce_soft_bf16(zd, lab, N, O, scale, d, loss, pred, labels_b=lb_d, lam=lam, smoothing=eps)
                eng.sync()
                dh = bits(d)
                ulps += check_soft(pkg, zb, labels, lb_h, lam, eps, scale, dh, loss.cpu().numpy(), pred.cpu().numpy())
                zi = zd.clone()
                eng.softmax_ce_soft_bf16(zi, lab, N, O, scale, zi, labels_b=lb_d, lam=lam, smoothing=eps)
                eng.sync()
                assert np.array_equal(bits(zi), dh)
    print(f"O = {O}: {ulps} values one ulp off over 18 cases")


@pytest.mark.parametrize("O", [1, 10, 256])
def test_soft_at_lam_1_eps_0_is_the_hard_loss(eng, pkg, O):
    """lam = 1 with eps = 0 gives pcnn_softmax_ce_bf16's dlogits, loss and pred bit for bit, for labels_b NULL, random or equal to
    labels, with NaN, -Inf and +Inf logits and labels >= O"""
    N = 300
    rng = np.random.default_rng(O)
    z = rng.normal(0, 3, (N, O)).astype(np.float32)
    z[5, O // 2] = np.nan
    z[11] = -np.inf
    z[12, 0] = np.inf
    z[13, O - 1] = -np.inf
    z[14] = np.inf
    zd = torch.from_numpy(pkg.f32_to_bf16_bits(z).view(np.int16)).to(DEV)
    labels = rng.integers(0, O, N).astype(np.uint8)
    labels[3] = 255
    lab = torch.from_numpy(labels).to(DEV)
    outs = lambda: (nan_buf(N, O), torch.zeros(N, dtype=torch.float32, device=DEV), torch.zeros(N, dtype=torch.int32, device=DEV))
    d0, l0, p0 = outs()
    eng.softmax_ce_bf16(zd, lab, N, O, 1.0 / N, d0, l0, p0)
    for lb in (None, torch.from_numpy(rng.integers(0, O, N).astype(np.uint8)).to(DEV), lab):
        d1, l1, p1 = outs()
        eng.softmax_ce_soft_bf16(zd, lab, N, O, 1.0 / N, d1, l1, p1, labels_b=lb, lam=1.0, smoothing=0.0)
        eng.sync()
        assert np.array_equal(bits(d1), bits(d0))
        assert np.array_equal(l1.cpu().numpy().view(np.uint32), l0.cpu().numpy().view(np.uint32))
        assert np.array_equal(p1.cpu().numpy(), p0.cpu().numpy())


# ------------------------------------------------------------------------------------------------ end to end
class MixedResNetGAP(ResNetGAP):
    """ResNetGAP whose loss is the soft-target one: forward(x, targets) runs the network, then pcnn_softmax_ce_soft_bf16 over its
    z into dz, loss and pred with the batcher's MixedLabels (or plain labels) and label smoothing EPS"""
    EPS = EPS

    def forward(self, x, targets, training=True):
        mixed = isinstance(targets, tuple)
        labels = targets.labels if mixed else targets
        super().forward(x, labels, training)
        self.eng.softmax_ce_soft_bf16(self.z, labels, self.NB, 10, 1.0 / self.NB, self.dz, self.loss, self.pred,
                                      labels_b=targets.labels_b if mixed else None, lam=targets.lam if mixed else 1.0,
                                      smoothing=self.EPS if training else 0.0)


def mnist_batcher(pkg, eng, golden, **k):
    return pkg.ImageBatcher(eng, golden["train_u8"].reshape(-1, 28, 28), golden["train_labels"], NB, row_pitch=32, image_rows=28, **k)


def test_resnet_gap_mixed(eng, pkg, golden):
    """The GAP ResNet fed by a batcher with shuffle, pad 2, mixup_alpha 0.2 and cutmix_alpha 1.0, trained against soft targets
    with label smoothing 0.1: the first 5 batches (x, both label vectors and the draws) and their dlogits on the device's own
    logits are bit-exact against the replay (one bf16 ulp near a rounding boundary), a fresh run reproduces the parameters after 5
    steps, the loss falls and test accuracy exceeds ACC_MIN.  Alphas 0 with eps 0 through the soft loss give, after 5 steps, the
    parameters of the hard-label run bit for bit."""
    make = lambda: MixedResNetGAP(eng, pkg, ResNetGAP.init_params())
    tests = pkg.ImageBatcher(eng, golden["test_u8"].reshape(-1, 28, 28), golden["test_labels"], NB, row_pitch=32, image_rows=28)
    train_u8 = golden["train_u8"].reshape(-1, 28, 28, 1)
    mixb = mnist_batcher(pkg, eng, golden, pad=2, shuffle=True, seed=SEED, mixup_alpha=ALPHAS[0], cutmix_alpha=ALPHAS[1])
    kinds = []

    def replayed(net, step, x, targets):
        kind, _, box, lam, _ = M.draws(SEED, 0, step, 28, 28, *ALPHAS)
        kinds.append(kind)
        assert isinstance(targets, pkg.MixedLabels) and (targets.kind, targets.lam, targets.box) == (kind, lam, box)
        mode = M.MIXUP if kind == "mixup" else M.CUTMIX
        wx, wl, wlb = M.batch(train_u8, step * NB, NB, mode, lam, box or (0, 0, 0, 0), 1, 2, 0, SEED, 0, labels=golden["train_labels"])
        xb = mixb.x.to_host()
        assert np.array_equal(xb[:, :, :28], wx.reshape(NB, 28, 28)) and (xb[:, :, 28:] == 0).all()
        assert np.array_equal(targets.labels.to_host(), wl) and np.array_equal(targets.labels_b.to_host(), wlb)
        net.forward(x, targets)
        eng.sync()
        zb = bits(net.z)
        check_soft(pkg, zb, wl, wlb, lam, EPS, 1.0 / NB, bits(net.dz), net.loss.cpu().numpy(), None)
        net.backward()

    loss_mix, acc_mix, _ = train(eng, pkg, golden, make, EPOCHS, batches=mixb, tests=tests, check_step=replayed)
    mixb.close()
    print(f"GAP ResNet on mixed batches (kinds of the first 5: {kinds}): mean loss {loss_mix[0]:.4f} -> {loss_mix[-1]:.4f}, "
          f"test accuracy {acc_mix:.4f} (threshold {ACC_MIN})")

    # alphas 0 and eps 0 through the soft loss: the hard-label run's parameters after 5 steps
    after5 = []
    for cls, eps in ((ResNetGAP, None), (MixedResNetGAP, 0.0)):
        plain = mnist_batcher(pkg, eng, golden, pad=2, shuffle=True, seed=SEED)
        net = cls(eng, pkg, ResNetGAP.init_params())
        if eps is not None:
            net.EPS = eps
        try:
            for s in range(5):
                x, lab = plain.batch(s)
                assert not isinstance(lab, tuple)
                net.forward(x, lab)
                net.backward()
                net.sgd(LR_STEP)
            eng.sync()
            after5.append(net.params())
        finally:
            net.close()
            plain.close()
    tests.close()
    assert same_bits(after5[0], after5[1])
    assert np.isfinite(loss_mix).all() and loss_mix[-1] < loss_mix[0]
    assert acc_mix > ACC_MIN
