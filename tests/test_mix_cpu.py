"""Mixed batches and soft targets without a GPU: mix_ref's CutMix box against torchvision's v2.CutMix.make_params, its soft target
and loss against torch's cross_entropy and autograd, the host draws of ImageBatcher (a function of (seed, epoch, step) alone, with
Beta(alpha, alpha) weights, an even MixUp / CutMix split and uniform centres), and the batcher's refusals of its new arguments
before any device call."""
import math
from unittest import mock

import numpy as np
import pytest
import torch
from torchvision.transforms import v2

import linear_ref as LR
import mix_ref as M

TINY = 1e-12


@pytest.mark.parametrize("H,W", [(28, 28), (24, 32), (5, 7), (1, 1)])
def test_cutmix_box_matches_torchvision(H, W):
    """box and lam_adjusted equal v2.CutMix.make_params' with its Beta sample and torch.randint patched to return lam and the
    centre, for lam in {0, tiny, 1/2, 1 - tiny, 1} and centres at the corners, the edges and the middle"""
    cm = v2.CutMix(alpha=1.0, num_classes=10)
    img = torch.zeros(2, 1, H, W)
    centres = {(0, 0), (W - 1, H - 1), (0, H - 1), (W - 1, 0), (W // 2, H // 2), (W // 3, 0)}
    for lam in (0.0, TINY, 0.5, 1.0 - TINY, 1.0):
        for r_x, r_y in sorted(centres):
            seq = iter([torch.tensor([r_x]), torch.tensor([r_y])])
            with mock.patch.object(cm._dist, "sample", return_value=torch.tensor([lam])), \
                    mock.patch("torch.randint", side_effect=lambda *a, **k: next(seq)):
                p = cm.make_params([img])
            box, lam_adj = M.cutmix_box(lam, r_x, r_y, H, W)
            assert box == p["box"] and lam_adj == p["lam_adjusted"], (lam, r_x, r_y, box, p)


def torch_soft(z, labels, labels_b, lam, eps, O):
    """torchvision's _mixup_label and cross_entropy's smoothing in fp32 torch: (m, q)"""
    oh = lambda y: torch.nn.functional.one_hot(torch.as_tensor(np.asarray(y).astype(np.int64)), O).float()
    m = oh(labels) if labels_b is None else oh(labels_b).mul_(1.0 - lam).add_(oh(labels).mul(lam))
    return m, m * (1.0 - eps) + eps / O


@pytest.mark.parametrize("O", [1, 10, 37, 256])
@pytest.mark.parametrize("lam", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("eps", [0.0, 0.1, 1.0])
def test_soft_reference_matches_torch(O, lam, eps):
    """q equals torch's fp32 target bit for bit; on finite rows the loss equals float64 cross_entropy(z, q) within 1e-12 and
    cross_entropy(z, m, label_smoothing=eps) within the fp32 rounding of q; g equals autograd's gradient of scale * sum loss up
    to the fp32 rounding of sum q"""
    N = 67
    rng = np.random.default_rng(O * 7 + int(lam * 10) + int(eps * 100))
    z = rng.normal(0, 3, (N, O))
    z[::5] = rng.integers(-2, 3, (len(z[::5]), O)) / 2.0
    labels, labels_b = rng.integers(0, O, N), rng.integers(0, O, N)
    labels_b[:9] = labels[:9]                                  # a row's two labels may coincide
    scale = 1.0 / N
    g, loss, pred, q = M.softmax_ce_soft_f64(z, labels, labels_b, lam, eps, scale)
    m_t, q_t = torch_soft(z, labels, labels_b, lam, eps, O)
    assert np.array_equal(q.view(np.uint32), q_t.numpy().view(np.uint32))
    zt = torch.tensor(z, requires_grad=True)
    ce = torch.nn.functional.cross_entropy(zt, q_t.double(), reduction="none")
    assert np.allclose(loss, ce.detach().numpy(), rtol=0, atol=1e-12)
    (ce.sum() * scale).backward()
    # autograd gives (p sum_t q_t - q) scale; the fp32 q sums to 1 only within its rounding, so that much of p scale is allowed
    off = np.abs(q.astype(np.float64).sum(axis=1, keepdims=True) - 1.0) * scale
    assert np.all(np.abs(g - zt.grad.numpy()) <= off + 1e-12)
    ls = torch.nn.functional.cross_entropy(torch.tensor(z), m_t.double(), label_smoothing=eps, reduction="none").numpy()
    assert np.allclose(loss, ls, rtol=1e-6, atol=1e-6)
    assert np.array_equal(pred, np.argmax(z, axis=1))


def test_soft_reference_reduces_to_the_hard_one():
    """lam = 1 with eps = 0 gives softmax_ce_f64's g, loss and pred exactly, for any labels_b and with NaN, -Inf, +Inf rows and
    labels >= O"""
    N, O = 40, 10
    rng = np.random.default_rng(3)
    z = rng.normal(0, 3, (N, O))
    z[1, 4] = np.nan
    z[2] = -np.inf
    z[3, 7] = np.inf
    z[4, 2] = -np.inf
    labels = rng.integers(0, O, N)
    labels[5] = O
    for labels_b in (None, rng.integers(0, O, N), np.full(N, 255)):
        g, loss, pred, _ = M.softmax_ce_soft_f64(z, labels, None if labels_b is None else labels_b, 1.0, 0.0, 0.5)
        if labels_b is not None and labels_b[0] == 255:
            continue                                           # a label_b >= O makes its row NaN, unlike the hard loss
        gh, lh, ph = LR.softmax_ce_f64(z, labels, 0.5)
        assert np.array_equal(g, gh, equal_nan=True) and np.array_equal(loss, lh, equal_nan=True) and np.array_equal(pred, ph)
    g, loss, _, _ = M.softmax_ce_soft_f64(z, labels, np.full(N, 255), 1.0, 0.0, 0.5)
    assert np.isnan(loss).all() and np.isnan(g).all()


def test_draws_depend_on_seed_epoch_and_step_alone(pkg):
    """the batcher's draws equal the replay's, repeat for the same (seed, epoch, step) and change with each of the three"""
    for seed in (0, 0x0123456789ABCDEF, (1 << 64) - 1):
        for epoch in (0, 1, (1 << 64) - 1):
            for step in (0, 1, 7):
                want = M.draws(seed, epoch, step, 28, 32, 0.2, 1.0)
                got = pkg.mix_draws(seed, epoch, step, 28, 32, 0.2, 1.0)
                assert got == (want[0], want[1], want[2], want[3] if want[0] == "cutmix" else None)
                assert M.draws(seed, epoch, step, 28, 32, 0.2, 1.0) == want
    lams = {M.draws(s, e, t, 28, 28, 0.2, 1.0)[1] for s in (0, 1) for e in (0, 1) for t in (0, 1)}
    assert len(lams) == 8


@pytest.mark.parametrize("mixup_alpha,cutmix_alpha", [(0.2, 1.0), (1.0, 0.0), (0.0, 0.4)])
def test_draw_statistics(mixup_alpha, cutmix_alpha):
    """over 20000 batches: the MixUp / CutMix split within 5 sigma of 1/2 (when both alphas > 0), each kind's lam mean and
    variance within 5 sigma of Beta(alpha, alpha)'s, and the CutMix centres uniform over W and H (every column and row count
    within 5 sigma)"""
    H, W, n = 24, 28, 20000
    d = [M.draws(0x5EED, e, s, H, W, mixup_alpha, cutmix_alpha) for e in range(20) for s in range(n // 20)]
    kinds = np.array([k == "cutmix" for k, *_ in d])
    if mixup_alpha > 0 and cutmix_alpha > 0:
        assert abs(kinds.mean() - 0.5) <= 5 * math.sqrt(0.25 / n)
    else:
        assert kinds.all() == (cutmix_alpha > 0) and kinds.any() == (cutmix_alpha > 0)
    for cut, alpha in ((False, mixup_alpha), (True, cutmix_alpha)):
        lam = np.array([x[1] for x, k in zip(d, kinds) if k == cut])
        if alpha == 0:
            assert lam.size == 0
            continue
        var = 1.0 / (4 * (2 * alpha + 1))                      # Beta(a, a): mean 1/2, variance 1 / (4 (2a + 1))
        mu4 = 3.0 * (alpha + 1) / (16 * (2 * alpha + 1) * (2 * alpha + 3))   # its fourth central moment
        assert abs(lam.mean() - 0.5) <= 5 * math.sqrt(var / lam.size)
        assert abs(lam.var() - var) <= 5 * math.sqrt((mu4 - var ** 2) / lam.size)
        assert lam.min() >= 0 and lam.max() <= 1
        if cut:
            c = np.array([x[4] for x, k in zip(d, kinds) if k])
            for vals, bins in ((c[:, 0], W), (c[:, 1], H)):
                counts = np.bincount(vals, minlength=bins)
                assert counts.size == bins
                p = 1.0 / bins
                assert np.all(np.abs(counts - lam.size * p) <= 5 * math.sqrt(lam.size * p * (1 - p)))
    print(f"alphas {mixup_alpha}/{cutmix_alpha}: CutMix share {kinds.mean():.4f}")


class NoDevice:
    """an engine whose every use fails the test: refusals must come first"""

    def __getattr__(self, name):
        raise AssertionError(f"device call {name} before the refusal")


@pytest.mark.parametrize("kw,msg", [
    (dict(mixup_alpha=-0.5), "mixup_alpha = -0.5: a finite alpha >= 0 is required"),
    (dict(mixup_alpha=float("nan")), "mixup_alpha = nan"),
    (dict(cutmix_alpha=float("inf")), "cutmix_alpha = inf"),
    (dict(cutmix_alpha="1"), "cutmix_alpha = 1: a finite alpha"),
    (dict(cutmix_alpha=1.0, labels=None), "needs labels to mix"),
])
def test_batcher_refusals_come_before_any_device_call(pkg, kw, msg):
    images, labels = np.zeros((16, 8, 8), np.uint8), np.zeros(16, np.uint8)
    args = dict(images=images, labels=labels, N=4)
    args.update(kw)
    with pytest.raises(pkg.PcnnError, match=msg):
        pkg.ImageBatcher(NoDevice(), **args)
