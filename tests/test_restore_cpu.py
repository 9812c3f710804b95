"""Host-side checks of image-to-image regression (no GPU): restore_ref's shuffle, unshuffle and loss replays pinned to torch's
pixel_shuffle / pixel_unshuffle and to mse_loss / l1_loss with float64 autograd, special values included; the domain and partition
of pcnn_pixel_shuffle_info; and pkg.psnr against its formula."""
import numpy as np
import pytest
import torch

import restore_ref as RR

F = torch.nn.functional


@pytest.mark.parametrize("N,H,W,C,r", [(1, 1, 1, 1, 1), (2, 3, 4, 1, 2), (1, 2, 3, 3, 3), (2, 2, 2, 8, 2), (1, 1, 2, 5, 4), (1, 2, 1, 2, 8)])
def test_shuffle_replays_are_torchs(N, H, W, C, r):
    rng = np.random.default_rng(N * 100 + C * 10 + r)
    x = rng.standard_normal((N, H, W, C * r * r)).astype(np.float32)
    want = F.pixel_shuffle(torch.from_numpy(x).permute(0, 3, 1, 2), r).permute(0, 2, 3, 1).numpy()
    assert np.array_equal(RR.shuffle(x, r), want)
    y = rng.standard_normal((N, H * r, W * r, C)).astype(np.float32)
    want = F.pixel_unshuffle(torch.from_numpy(y).permute(0, 3, 1, 2), r).permute(0, 2, 3, 1).numpy()
    assert np.array_equal(RR.unshuffle(y, r), want)
    assert np.array_equal(RR.unshuffle(RR.shuffle(x, r), r), x) and np.array_equal(RR.shuffle(RR.unshuffle(y, r), r), y)
    if r > 1 and C > 1:          # TensorFlow's depth_to_space is a different permutation
        assert not np.array_equal(RR.depth_to_space(x, r), RR.shuffle(x, r))


def _operands(rng, P, C, special):
    p = rng.standard_normal((P, C)).astype(np.float32)
    t = rng.standard_normal((P, C)).astype(np.float32)
    if special:
        pv = [0.0, -0.0, 0.0, np.nan, np.inf, -np.inf, 1.0]
        tv = [0.0, 0.0, -0.0, 0.0, 1.0, 1.0, np.nan]
        p.reshape(-1)[:len(pv)], t.reshape(-1)[:len(tv)] = pv, tv
    return RR.bf16_bits(p), RR.bf16_bits(t)


@pytest.mark.parametrize("mode", [RR.MSE, RR.L1])
@pytest.mark.parametrize("P,C,special", [(300, 1, False), (97, 3, True), (64, 16, True), (5, 130, False)])
def test_loss_replay_is_torchs_float64_autograd(mode, P, C, special):
    rng = np.random.default_rng(P + C + mode)
    pb, tb = _operands(rng, P, C, special)
    scale = 1.0 / (P * C)
    g, loss = RR.loss_replay(pb, tb, C, mode, scale)
    p64 = torch.from_numpy(RR.bits_f32(pb).astype(np.float64)).requires_grad_(True)
    t64 = torch.from_numpy(RR.bits_f32(tb).astype(np.float64))
    lt = (F.mse_loss if mode == RR.MSE else F.l1_loss)(p64, t64)
    lt.backward()
    want, got = p64.grad.numpy(), RR.bits_f32(g).astype(np.float64).reshape(P, C)
    fin = np.isfinite(want)
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[~fin & ~np.isnan(want)], want[~fin & ~np.isnan(want)])
    assert np.all(np.abs(got[fin] - want[fin]) <= 2 ** -8 * np.abs(want[fin]) + 1e-45)
    assert np.array_equal(np.signbit(got[want == 0]), np.signbit(want[want == 0]))       # -0 (MSE at d = -0) and +0 kept apart
    mean = loss.astype(np.float64).sum() / (P * C)
    ref = lt.item()
    if special:
        assert np.isnan(mean) and np.isnan(ref)
    else:
        assert abs(mean - ref) <= 1e-5 * abs(ref)
        # each pixel's loss against its float64 sum
        d = RR.bits_f32(pb).astype(np.float64).reshape(P, C) - RR.bits_f32(tb).astype(np.float64).reshape(P, C)
        per = (d * d if mode == RR.MSE else np.abs(d)).sum(1)
        assert np.all(np.abs(loss - per) <= (C + 2) * 2 ** -24 * per)


def test_loss_special_values_as_stated():
    """include/pcnn.h's special values: MSE -0 at d = -0, NaN at NaN, +-Inf at +-Inf, and +Inf where a finite p - t overflows fp32
    (float64 autograd stays finite there); L1 +0 at +-0 and at NaN (terms NaN)"""
    p = np.array([[0.0, -0.0, np.nan, np.inf, -np.inf, 2.0, 3e38]], np.float32)
    t = np.array([[0.0, 0.0, 0.0, 1.0, 1.0, 1.0, -3e38]], np.float32)
    g, loss = RR.loss_replay(RR.bf16_bits(p), RR.bf16_bits(t), 7, RR.MSE, 0.5)
    assert list(g.reshape(-1)) == [0x0000, 0x8000, 0x7FFF, 0x7F80, 0xFF80, 0x3F80, 0x7F80] and np.isnan(loss[0])
    g, loss = RR.loss_replay(RR.bf16_bits(p), RR.bf16_bits(t), 7, RR.L1, 0.5)
    assert list(g.reshape(-1)) == [0x0000, 0x0000, 0x0000, 0x3F00, 0xBF00, 0x3F00, 0x3F00] and np.isnan(loss[0])


def test_loss_replay_reads_the_first_c_channels_of_a_pitched_target():
    rng = np.random.default_rng(4)
    pb, tb = _operands(rng, 50, 3, False)
    wide = rng.integers(0, 0x7F00, (50, 8)).astype(np.uint16)
    wide[:, :3] = tb
    for mode in (RR.MSE, RR.L1):
        a, b = RR.loss_replay(pb, tb, 3, mode, 0.01), RR.loss_replay(pb, wide, 3, mode, 0.01, target_stride=8)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_pixel_shuffle_info_partition(pkg):
    for N, H, W, C, r in [(16, 128, 128, 3, 2), (16, 64, 64, 3, 4), (16, 48, 48, 64, 2), (128, 28, 28, 64, 2), (1, 1, 1, 1, 1),
                          (2, 3, 5, 256, 8), (1, 7, 9, 24, 3), (3, 2, 2, 1000, 5)]:
        for unshuffle in (False, True):
            Hs, Ws = (H * r, W * r) if unshuffle else (H, W)
            info = pkg.pixel_shuffle_info(N, Hs, Ws, C, r, unshuffle=unshuffle)
            assert info["vec"] == (8 if C % 8 == 0 else 1) and info["threads"] == 256
            P, Cc = info["tile_pixels"], info["chunk_channels"]
            assert 1 <= P and Cc * r * r * P <= 4096 and Cc % info["vec"] == 0
            assert Cc == C if C * r * r <= 4096 else Cc < C
            assert info["grid"] == -(-N * H * W // P) * -(-C // Cc)
            assert info["smem"] <= 48 * 1024


def test_pixel_shuffle_info_refusals(pkg):
    cases = [((0, 4, 4, 8, 2), {}, "N = 0"), ((1, 0, 4, 8, 2), {}, "H = 0"), ((1, 4, 4, 0, 2), {}, "C = 0"), ((1, 4, 4, 8, 0), {}, "r = 0"),
             ((1, 4, 4, 8, 9), {}, "r = 9"), ((1, 6, 4, 8, 4), {"unshuffle": True}, "multiples of r"),
             ((1, 4, 6, 8, 4), {"unshuffle": True}, "multiples of r"), ((64, 1024, 1024, 64, 2), {}, "2\\^31 - 1"),
             ((4096, 1024, 1024, 1, 1), {"unshuffle": True}, "2\\^31 - 1")]
    for args, kw, msg in cases:
        with pytest.raises(pkg.PcnnError, match=msg):
            pkg.pixel_shuffle_info(*args, **kw)
    pkg.pixel_shuffle_info(1, 6, 4, 8, 4)                       # the shuffle takes any H and W
    pkg.pixel_shuffle_info(31, 1024, 1024, 64, 1)               # 31 * 2^26 elements fit; 2^31 would not
    out = (pkg._lib._ll * 6)()
    with pytest.raises(pkg.PcnnError, match="unshuffle = 2"):
        pkg._lib.check("pcnn_pixel_shuffle_info", pkg.lib().pcnn_pixel_shuffle_info(1, 4, 4, 8, 2, 2, out))


def test_psnr_formula(pkg):
    rng = np.random.default_rng(7)
    t = rng.random((5, 28, 28, 1))
    p = t + rng.standard_normal(t.shape) * 0.05
    want = np.mean([10 * np.log10(1.0 / np.mean((p[i] - t[i]) ** 2)) for i in range(5)])
    assert abs(pkg.psnr(p, t) - want) <= 1e-12 * abs(want)
    assert abs(pkg.psnr(p * 255, t * 255, data_range=255.0) - want) <= 1e-9 * abs(want)
    assert pkg.psnr(t, t) == np.inf
    with pytest.raises(pkg.PcnnError, match="differ"):
        pkg.psnr(p[:, :, :, 0], t)
