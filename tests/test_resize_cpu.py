"""Resized batches on the host (resize_ref.py, pcnn_augment_resized_u8_bf16_info): the replay's resample bit for bit against torch's
uint8 antialiased bilinear resize, the eval window against torchvision's Resize + CenterCrop, the box rule against
v2.RandomResizedCrop.make_params with the draws injected, the boxes E changes against torch's exp, box statistics, counter
domains, and the info query with every refusal, also in a process without a GPU."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torchvision.transforms.v2 as v2
import torchvision.transforms.v2.functional as TF

import augment_ref as A
import resize_ref as RR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 0x0123456789ABCDEF


def chw(img):
    return torch.from_numpy(np.ascontiguousarray(img)).permute(2, 0, 1).contiguous()


def hwc(t):
    return t.permute(1, 2, 0).numpy()


def random_shapes(count, seed):
    """(H, W, C, h, w): sides 1 .. 500, every downscale within the 16x domain, one axis unchanged in every fifth case"""
    rng = np.random.default_rng(seed)
    for k in range(count):
        C = int(rng.choice([1, 3, 4]))
        H, W = (int(v) for v in rng.integers(1, 501, 2))
        h, w = int(rng.integers(-(-H // 16), 501)), int(rng.integers(-(-W // 16), 501))
        if k % 5 == 1:
            w = W
        elif k % 5 == 3:
            h = H
        yield H, W, C, h, w, rng


def test_resample_is_torch_resize():
    """the replay's resample equals TF.resize(antialias=True) and TF.resized_crop on uint8 CPU tensors, bit for bit"""
    n = 0
    for H, W, C, h, w, rng in random_shapes(300, 1):
        img = rng.integers(0, 256, (H, W, C), dtype=np.uint8)
        want = hwc(TF.resize(chw(img), [h, w], antialias=True))
        assert np.array_equal(RR.resample(img, h, w), want), (H, W, C, h, w)
        t, l = int(rng.integers(0, H)), int(rng.integers(0, W))
        bh, bw = int(rng.integers(1, H - t + 1)), int(rng.integers(1, W - l + 1))
        want = hwc(TF.resized_crop(chw(img), t, l, bh, bw, [h, w], antialias=True))
        assert np.array_equal(RR.resample(img[t:t + bh, l:l + bw], h, w), want), (H, W, C, t, l, bh, bw, h, w)
        n += 1
    assert n == 300


@pytest.mark.parametrize("H,W,size,crop", [(37, 53, 30, 24), (53, 37, 30, 28), (64, 64, 72, 56), (256, 256, 256, 224),
                                           (320, 240, 256, 224), (240, 320, 224, 224), (28, 28, 20, 28), (28, 28, 24, 32),
                                           (5, 90, 7, (11, 4)), (90, 5, 3, (2, 9)), (1, 1, 1, 3)])
def test_eval_window_is_resize_center_crop(pkg, H, W, size, crop):
    """Resize(size) + CenterCrop(crop), a crop larger than the resized image included, equals the replay; the info query gives the
    same resized size and window"""
    rng = np.random.default_rng([H, W, size])
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    ch, cw = (crop, crop) if isinstance(crop, int) else crop
    want = hwc(v2.Compose([v2.Resize(size, antialias=True), v2.CenterCrop((ch, cw))])(chw(img)))
    assert np.array_equal(RR.eval_image(img, size, ch, cw), want)
    info, _ = pkg.augment_resized_info(8, H, W, 3, 0, 8, ch, cw, mode=pkg.RESIZE_EVAL, resize_size=size)
    Rh, Rw = RR.resized_size(H, W, size)
    assert (info["Rh"], info["Rw"], info["ty"], info["tx"]) == (Rh, Rw, RR.anchor(Rh, ch), RR.anchor(Rw, cw))
    if (H, W, size) == (37, 53, 30):
        assert (Rh, Rw) == (30, 42)


def torch_exp(x):
    return torch.exp(torch.from_numpy(np.asarray(x, np.float32))).numpy()


BOX_CASES = [  # (H, W, scale, ratio): the defaults, fallbacks on every side, s1 > 1, a one-pixel side
    (224, 224, (0.08, 1.0), (3 / 4, 4 / 3)),
    (256, 320, (0.08, 1.0), (3 / 4, 4 / 3)),
    (28, 28, (0.35, 1.0), (3 / 4, 4 / 3)),
    (40, 10, (0.9, 1.0), (3 / 4, 4 / 3)),          # W / H < r0: the fallback narrows h
    (10, 40, (0.9, 1.0), (3 / 4, 4 / 3)),          # W / H > r1: the fallback narrows w
    (30, 30, (2.0, 5.0), (3 / 4, 4 / 3)),          # nothing fits: the whole image
    (17, 29, (0.5, 1.5), (0.2, 5.0)),
    (1, 64, (0.01, 1.0), (10.0, 80.0)),
]


@pytest.mark.parametrize("H,W,scale,ratio", BOX_CASES)
def test_box_rule_is_make_params(monkeypatch, pkg, H, W, scale, ratio):
    """make_params, with its uniforms replaced by the device's s and lr and its randints by umulhi of the device's words, gives the
    replay's box when the replay takes torch's float32 exp; with E, any box that differs is one where E and exp differ"""
    i = np.arange(400, dtype=np.uint64) * np.uint64(7919)
    s, lr, wt, wl = RR.box_draws(i, scale, ratio, SEED, 3)
    got = RR.choose_box(H, W, s, lr, wt, wl, ratio, exp=torch_exp)
    dev = RR.choose_box(H, W, s, lr, wt, wl, ratio)
    t = v2.RandomResizedCrop((8, 8), scale=scale, ratio=ratio, antialias=True)
    queue, words = [], []
    monkeypatch.setattr(torch.Tensor, "uniform_", lambda self, a, b: self.fill_(float(queue.pop(0))))
    monkeypatch.setattr(torch, "randint", lambda lo, hi, size: torch.tensor([int(RR.umulhi(words.pop(0), hi))]))
    fallbacks = changed = 0
    for k in range(len(i)):
        queue[:] = [v for a in range(RR.ATTEMPTS) for v in (s[k, a], lr[k, a])]
        words[:] = [wt[k], wl[k]]
        p = t.make_params([torch.zeros(3, H, W)])
        box = (p["top"], p["left"], p["height"], p["width"])
        assert box == tuple(int(v[k]) for v in got[:4]), (k, box)
        fallbacks += got[4][k] < 0
        if box != tuple(int(v[k]) for v in dev[:4]):
            changed += 1
            assert torch_exp(lr[k]).tolist() != RR.exp_f32(lr[k]).tolist()
    assert changed <= 2
    assert pkg.augment_resized_info(8, H, W, 3, 0, 8, H, W, scale=scale, ratio=ratio)[0]["fallback"] == RR.fallback(H, W, ratio)
    if scale[0] > 1.5 or (scale[0] > 0.8 and not ratio[0] <= W / H <= ratio[1]):
        assert fallbacks > 0


def test_log_ratio_is_torch_log():
    """log r0 and log r1, rounded to fp32 on the host, are torchvision's torch.log(torch.tensor(ratio))"""
    rng = np.random.default_rng(5)
    for ratio in [(3 / 4, 4 / 3), (0.5, 2.0), (1.0, 1.0)] + [tuple(sorted(rng.uniform(0.05, 20.0, 2).tolist())) for _ in range(500)]:
        l0 = RR.box_constants((0.5, 1.0), ratio)[2]
        l1 = RR.box_constants((0.5, 1.0), ratio[::-1])[2]
        want = torch.log(torch.tensor(ratio)).numpy()
        assert want.dtype == np.float32 and (l0, l1) == (want[0], want[1]), ratio


def test_boxes_e_changes_over_a_million_draws():
    """how many of 10^6 images' boxes change when E replaces torch's float32 exp (224 x 224, the default scale and ratio)"""
    i = np.arange(1_000_000, dtype=np.uint64)
    s, lr, wt, wl = RR.box_draws(i, (0.08, 1.0), (3 / 4, 4 / 3), SEED, 0)
    e = RR.choose_box(224, 224, s, lr, wt, wl, (3 / 4, 4 / 3))
    t = RR.choose_box(224, 224, s, lr, wt, wl, (3 / 4, 4 / 3), exp=torch_exp)
    changed = int(np.any(np.stack(e[:4]) != np.stack(t[:4]), axis=0).sum())
    differ = int((RR.exp_f32(lr) != torch_exp(lr)).sum())
    print(f"E and torch's exp differ on {differ} of {lr.size} draws of lr; {changed} of {len(i)} boxes change")
    assert changed <= 20


def test_box_statistics():
    """with every first attempt fitting (1000 x 1000, scale (0.08, 0.5)), the area fraction and log(w / h) of 10^5 boxes have the
    means and variances of U(0.08, 0.5) and U(log 3/4, log 4/3) within 5 sigma, and top / (H - h) is uniform"""
    n = 100_000
    lo, hi = 0.08, 0.5
    top, left, h, w, att = RR.boxes(np.arange(n, dtype=np.uint64), 1000, 1000, (lo, hi), (3 / 4, 4 / 3), SEED, 9)
    assert (att == 0).all()
    a = h * w / 1e6
    la, lb = math.log(3 / 4), math.log(4 / 3)
    r = np.log(w / h)
    for v, p, q in ((a, lo, hi), (r, la, lb)):
        var = (q - p) ** 2 / 12
        assert abs(v.mean() - (p + q) / 2) < 5 * math.sqrt(var / n) + 2e-4
        assert abs(v.var() - var) < 5 * math.sqrt(var * var * 0.8 / n) + 2e-4      # Var of (x - mu)^2 for a uniform is 0.8 var^2
    f = top / np.maximum(1000 - h, 1)
    assert abs(f.mean() - 0.5) < 5 * math.sqrt(1 / 12 / n)
    assert 0 <= top.min() and (top + h).max() <= 1000 and (left + w).max() <= 1000


def test_box_counters_are_their_own():
    """word 1 of a box counter, for any index below 2^56 and block 0..5, is >= 0xC8000000: above every permutation round's word
    (0xC0000000 | r), with bit 30 set where a crop counter's is clear (i < 2^62), and bit 31 set where a dropout counter's is clear"""
    i = np.array([0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 40 + 17, 2 ** 56 - 1], np.uint64)
    words = np.concatenate([RR.box_counters(i, k, 0)[1] for k in range(RR.ATTEMPTS // 2 + 1)]).astype(np.uint64)
    assert (words >= 0xC8000000).all() and (words <= 0xCDFFFFFF).all()
    perm = np.array([A.round_counters(np.zeros(1), r, 0)[1] for r in range(A.ROUNDS)], np.uint64)
    assert perm.max() < 0xC8000000
    crop = A.crop_counters(np.array([0, 2 ** 62 - 1], np.uint64), 0)[1]
    assert ((crop & np.uint64(0x40000000)) == 0).all() and ((words & np.uint64(0x40000000)) != 0).all()
    assert ((words & np.uint64(0x80000000)) != 0).all()
    pairs = {(int(w0), int(w1)) for k in range(RR.ATTEMPTS // 2 + 1) for w0, w1 in zip(*RR.box_counters(i, k, 0)[:2])}
    assert len(pairs) == len(i) * (RR.ATTEMPTS // 2 + 1)


OK = dict(n=64, H=32, W=32, C=3, first=0, N=8, H_out=24, W_out=24, mode=1, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3), resize_size=28,
          shuffle=1, flip=1, C_out=8, row_pitch=0, image_rows=0, mean=None, std=None)
F = "pcnn_augment_resized_u8_bf16_info: "
REFUSALS = [
    (dict(n=0), F + "n = 0, N = 8, H = 32, W = 32, H_out = 24, W_out = 24: each must be >= 1"),
    (dict(W_out=0), "W_out = 0: each must be >= 1"),
    (dict(first=57), "first = 57, N = 8: 0 <= first and first \\+ N <= n = 64 are required"),
    (dict(n=(1 << 56) + 1, H=1, W=1, C=1), "n = 72057594037927937: n <= 2\\^56 is required"),
    (dict(C=5, C_out=8), "C = 5: 1 <= C <= 4 is required"),
    (dict(C_out=2), "C_out = 2: C = 3 <= C_out <= 8 is required"),
    (dict(shuffle=2), "shuffle = 2, flip = 1: each must be 0 or 1"),
    (dict(flip=-1), "shuffle = 1, flip = -1: each must be 0 or 1"),
    (dict(mode=0), "mode = 0: 1 \\(train\\) or 2 \\(eval\\) is required"),
    (dict(mode=3), "mode = 3"),
    (dict(H=1 << 16, W=1 << 14, C=2, N=1), "H W C = 2147483648: one image must fit the 32-bit range"),
    (dict(n=1 << 41, H=1 << 12, W=1 << 10, C=1), "the dataset must be below 2\\^62 bytes"),
    (dict(H_out=16385), "H_out = 16385, W_out = 24: each must be <= 16384"),
    (dict(row_pitch=188), "row_pitch = 188: 0 \\(W_out C_out = 192 rounded up to 8\\) or a multiple of 8 >= W_out C_out is required"),
    (dict(image_rows=23), "image_rows = 23: 0 \\(H_out\\) or >= H_out = 24 is required"),
    (dict(row_pitch=1 << 30, image_rows=1 << 30), "x must be below 2\\^62 bytes"),
    (dict(mean=(0.0, float("nan"), 0.0)), "mean\\[1\\] = nan: a finite mean is required"),
    (dict(std=(1.0, 0.0, 1.0)), "std\\[1\\] = 0: a finite std > 0 is required"),
    (dict(scale=(float("nan"), 1.0)), "scale = \\(nan, 1\\), ratio = \\(0.75, 1.33333\\): each must be finite and within fp32's normal"),
    (dict(scale=(0.0, 1.0)), "scale = \\(0, 1\\)"),
    (dict(scale=(-0.5, 1.0)), "scale = \\(-0.5, 1\\)"),
    (dict(scale=(0.5, float("inf"))), "each must be finite and within"),
    (dict(ratio=(0.0, 1.0)), "ratio = \\(0, 1\\): each must be finite"),
    (dict(ratio=(1.0, 1e39)), "each must be finite and within"),
    (dict(scale=(0.9, 0.5)), "scale = \\(0.9, 0.5\\), ratio = \\(0.75, 1.33333\\): each range must be \\(min, max\\)"),
    (dict(ratio=(2.0, 1.0)), "each range must be \\(min, max\\)"),
    (dict(H=1, W=1, ratio=(3.0, 4.0)), "ratio = \\(3, 4\\): the central fallback crop of a 1 x 1 image is empty"),
    (dict(mode=2, resize_size=0), "resize_size = 0: 1 <= resize_size <= 16384 is required"),
    (dict(mode=2, resize_size=-3), "resize_size = -3"),
    (dict(mode=2, H=1, W=8, resize_size=4096), "resize_size = 4096: the longer resized side, 32768, must be <= 16384"),
    (dict(H=32, W=400, W_out=24), "32 x 400 to 24 x 24: the whole image needs 5 x 35 taps, at most 33 per axis"),
    (dict(mode=2, H=400, W=400, resize_size=24), "400 x 400 to 24 x 24: the whole image needs 35 x 35 taps"),
    (dict(H=512, W=8192, C=4, H_out=512, W_out=8192), "W_out C = 8192 x 4: one output row of the whole image needs \\d+ bytes of shared"),
    (dict(H=3584, W=3584, C=4, H_out=224, W_out=224), "W_out C = 224 x 4: one output row of the whole image needs 48032 bytes of shared "
                                                      "memory, at most 46928 are available"),
]


@pytest.mark.parametrize("change,msg", REFUSALS)
def test_info_refusals(pkg, change, msg):
    with pytest.raises(pkg.PcnnError, match=msg):
        pkg.augment_resized_info(**dict(OK, **change))


def test_refusals_in_a_process_without_a_gpu(pkg):
    """the query answers and refuses with the same messages where no GPU is visible"""
    cases = [OK] + [dict(OK, **c) for c, _ in REFUSALS]
    code = ("import json, math, pcnn_loader; pkg = pcnn_loader.load(); out = []\n"
            f"for a in json.loads({json.dumps(json.dumps(cases))}):\n"
            "    try:\n        out.append(pkg.augment_resized_info(**a)[0])\n"
            "    except pkg.PcnnError as e:\n        out.append(e.msg)\n"
            "print(json.dumps(out))")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = json.loads(subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, check=True).stdout)
    info = pkg.augment_resized_info(**OK)[0]
    info["fallback"] = list(info["fallback"])
    assert out[0] == info
    for a, msg in zip(cases[1:], out[1:]):
        with pytest.raises(pkg.PcnnError) as e:
            pkg.augment_resized_info(**a)
        assert msg == e.value.msg


def dynamic_bytes(info, rpc, H, H_out, W_out, C):
    """the dynamic shared memory of a unit of rpc rows (pcnn.h): x0 / xn, y0 / yn, both tap tables and rows_cap source rows"""
    up = lambda v: -(-v // 16) * 16
    scale = H / H_out
    cap = int(min(H, math.floor(scale * (rpc - 1) + 2 * max(scale, 1.0) + 1.0) + 2))
    return up(8 * W_out) + up(8 * rpc) + up(2 * W_out * info["taps_x"]) + up(2 * rpc * info["taps_y"]) + cap * W_out * C


@pytest.mark.parametrize("H_out,W_out,H,W,C,mode,rpc", [(224, 224, 256, 256, 3, 1, 32), (28, 28, 28, 28, 1, 1, 28), (56, 56, 64, 64, 3, 1, 32),
                                                        (224, 224, 480, 640, 3, 1, 26), (224, 224, 500, 375, 3, 1, 25),
                                                        (224, 224, 600, 800, 3, 1, 20), (224, 224, 2048, 2048, 4, 1, 3), (224, 224, 3000, 3000, 4, 1, 1)])
def test_info_launch(pkg, H_out, W_out, H, W, C, mode, rpc):
    """rows per CTA is the largest <= min(H_out, 32) whose worst-case dynamic shared memory, added to the kernel's static shared
    memory, fits the 48 KB a launch gets without an opt-in"""
    info, _ = pkg.augment_resized_info(1024, H, W, C, 0, 256, H_out, W_out, mode=mode, C_out=8)
    budget = 48 * 1024 - info["static_smem"]
    assert info["static_smem"] >= 2 * 4 * 256 and info["static_smem"] % 16 == 0
    assert info["rows_per_cta"] == rpc and info["smem"] == dynamic_bytes(info, rpc, H, H_out, W_out, C) <= budget
    if rpc < min(H_out, 32):
        assert dynamic_bytes(info, rpc + 1, H, H_out, W_out, C) > budget
    assert info["row_blocks"] == -(-H_out // rpc) and info["grid"] == 256 * info["row_blocks"]
    assert info["taps_y"] == 2 * math.ceil(max(H / H_out, 1)) + 1 and info["vec"] == 8


def test_batcher_refuses_before_touching_the_engine(pkg):
    img = np.zeros((16, 8, 8, 3), np.uint8)
    lab = np.zeros(16, np.uint8)
    with pytest.raises(pkg.PcnnError, match="crop_size = 6 with pad = 2: a resized batch takes no padding"):
        pkg.ImageBatcher(None, img, lab, 4, pad=2, crop_size=6)
    with pytest.raises(pkg.PcnnError, match="crop_size = 6 with mixup_alpha or cutmix_alpha > 0: resized batches are not mixed"):
        pkg.ImageBatcher(None, img, lab, 4, crop_size=6, mixup_alpha=0.2)
    with pytest.raises(pkg.PcnnError, match="crop_size = 6 with mixup_alpha"):
        pkg.ImageBatcher(None, img, lab, 4, crop_size=6, cutmix_alpha=1.0)
    with pytest.raises(pkg.PcnnError, match="resize_size = 8 without crop_size"):
        pkg.ImageBatcher(None, img, lab, 4, resize_size=8)
    with pytest.raises(pkg.PcnnError, match="scale = \\(0.9, 0.5\\)"):
        pkg.ImageBatcher(None, img, lab, 4, crop_size=6, scale=(0.9, 0.5))
    with pytest.raises(pkg.PcnnError, match="resize_size = 0: 1 <= resize_size"):
        pkg.ImageBatcher(None, img, lab, 4, crop_size=6, resize_size=0)
    with pytest.raises(pkg.PcnnError, match="8 x 400 to 8 x 8: the whole image needs 3 x 101 taps"):
        pkg.ImageBatcher(None, np.zeros((16, 8, 400, 3), np.uint8), lab, 4, crop_size=(8, 8))
