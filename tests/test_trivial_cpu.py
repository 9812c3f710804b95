"""TrivialAugmentWide and RandomErasing on the host (trivial_ref.py, pcnn_augment_trivial_u8_bf16_info): the library's table against
torchvision's formulas, the replay's ops bit for bit against torchvision's _apply_op where pcnn.h calls them exact, the measured and
confined disagreement where the fp32 order is the device's own, the erase box against RandomErasing.get_params with the draws
injected, draw statistics, counter domains, and every refusal of the info query and the batcher, also in a process without a GPU."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torchvision.transforms as T
from torchvision.transforms import InterpolationMode
from torchvision.transforms import autoaugment as aa

import augment_ref as A
import resize_ref as RR
import trivial_ref as TR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 0x0123456789ABCDEF
EXACT = ("Identity", "Brightness", "Color", "Contrast", "Posterize", "Solarize", "AutoContrast", "Equalize")
GEOMETRIC = ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate")
MODES = {TR.NEAREST: InterpolationMode.NEAREST, TR.BILINEAR: InterpolationMode.BILINEAR}


def torch_op(img, op, b, sign, interp=TR.NEAREST):
    """torchvision's _apply_op on uint8 [h][w][C] with the magnitude of (op, bin, sign) from _augmentation_space"""
    mag = TR.magnitude(TR.magnitudes(), op, b, sign)
    t = torch.from_numpy(np.ascontiguousarray(img)).permute(2, 0, 1).contiguous()
    return aa._apply_op(t, TR.OPS[op], mag, interpolation=MODES[interp], fill=None).permute(1, 2, 0).numpy()


def images(seed, count, max_side=64):
    """random crops, C 1 or 3, with flat, one-valued and two-valued ones among them"""
    rng = np.random.default_rng(seed)
    for k in range(count):
        C = int(rng.choice([1, 3]))
        h, w = (int(v) for v in rng.integers(1, max_side + 1, 2))
        kind = k % 5
        if kind == 0:
            img = np.full((h, w, C), int(rng.integers(0, 256)), np.uint8)
        elif kind == 1:
            img = np.where(rng.random((h, w, C)) < 0.5, int(rng.integers(0, 256)), int(rng.integers(0, 256))).astype(np.uint8)
        elif kind == 2:
            img = np.where(rng.random((h, w, 1)) < 0.01, 255, 7).astype(np.uint8).repeat(C, -1)
        else:
            img = rng.integers(0, 256, (h, w, C), dtype=np.uint8)
        yield img


@pytest.mark.parametrize("h,w", [(224, 224), (256, 256), (28, 32), (32, 32), (1, 1), (3, 200), (17, 5)])
def test_table_is_torchvision(pkg, h, w):
    """the library's host table, built in C, is the one torchvision's Python formulas give for every (op, bin, sign)"""
    _, tab, _ = pkg.augment_trivial_info(8, h, w, 3, 0, 8)
    want = TR.table(h, w)
    assert np.array_equal(tab.view(np.uint32), want.view(np.uint32))


def test_magnitudes_are_the_libraries():
    """the magnitudes pcnn.h states (Rotate's 4.5 b, Solarize's 255 - 8.5 b, Posterize's 8 - round(b / 5)) are _augmentation_space's"""
    m = TR.magnitudes()
    b = np.arange(31)
    assert np.array_equal(m["Rotate"][0], (np.float32(4.5) * b.astype(np.float32)).astype(np.float64))
    assert np.array_equal(m["Solarize"][0], (np.float32(255) - np.float32(8.5) * b.astype(np.float32)).astype(np.float64))
    assert np.array_equal(m["Posterize"][0], 8 - np.rint(b.astype(np.float32) / np.float32(5)))
    assert [s for _, s in m.values()] == [op in TR.SIGNED for op in TR.OPS]


@pytest.mark.parametrize("op", EXACT + ("TranslateX", "TranslateY"))
def test_exact_ops_are_apply_op(op):
    """every bin and sign of the exact ops (and NEAREST integer translations) on random crops, C 1 and 3, 1 x 1 .. 64 x 64 and a
    few up to 256 x 256, flat, one- and two-valued ones included: the replay is torchvision's _apply_op bit for bit"""
    k = TR.OPS.index(op)
    imgs = list(images(k, 12)) + list(images(100 + k, 2, 256))
    for img in imgs:
        h, w = img.shape[:2]
        tab = TR.table(h, w)
        for b in range(31):
            for s in range(2):
                want = torch_op(img, k, b, s)
                got = TR.apply_op(img, k, tab[k, b, s], TR.NEAREST)
                assert np.array_equal(got, want), (op, b, s, img.shape)


def test_contrast_domain_at_256_squared():
    """at 256 x 256 (the largest crop) a white image's fp32 mean is exact: the sum 256^2 255 < 2^24"""
    img = np.full((256, 256, 3), 255, np.uint8)
    k = TR.OPS.index("Contrast")
    tab = TR.table(256, 256)
    for b in (0, 15, 30):
        assert np.array_equal(TR.apply_op(img, k, tab[k, b, 1], TR.NEAREST), torch_op(img, k, b, 1))


def neighbours(img, ix, iy):
    """the source values at the 3 x 3 neighbourhood of the rounded coordinates, 0 outside: [h][w][9][C]"""
    h, w, C = img.shape
    out = []
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            fy, fx = np.rint(iy) + dy, np.rint(ix) + dx
            ok = (fx >= 0) & (fx < w) & (fy >= 0) & (fy < h)
            out.append(np.where(ok[..., None], img[np.where(ok, fy, 0).astype(int), np.where(ok, fx, 0).astype(int)], 0))
    return np.stack(out, 2)


@pytest.mark.parametrize("interp", [TR.NEAREST, TR.BILINEAR])
def test_order_dependent_ops_agree_within_allowance(interp):
    """Shear, Rotate, Sharpness and every bilinear op evaluate in the device's fp32 order (pcnn.h); against torchvision's CPU order
    the rate of differing pixels per 10^6 is printed and bounded, and every difference is confined: NEAREST takes a neighbouring
    source pixel, a rounding differs by 1"""
    ops = GEOMETRIC + ("Sharpness",) if interp == TR.NEAREST else GEOMETRIC
    total = 0
    bad = {}
    for img in images(77 + interp, 10, 96):
        h, w, C = img.shape
        tab = TR.table(h, w)
        for op in ops:
            k = TR.OPS.index(op)
            for b in range(0, 31, 3):
                for s in range(2):
                    want = torch_op(img, k, b, s, interp).astype(np.int64)
                    got = TR.apply_op(img, k, tab[k, b, s], interp).astype(np.int64)
                    diff = np.any(got != want, -1)
                    total += h * w
                    bad[op] = bad.get(op, 0) + int(diff.sum())
                    if not diff.any():
                        continue
                    if interp == TR.NEAREST and op != "Sharpness":
                        ix, iy = TR.grid_coords(h, w, tab[k, b, s])
                        nb = neighbours(img, ix, iy).astype(np.int64)
                        assert np.all(np.any(np.all(nb == want[:, :, None, :], -1), -1)[diff]), (op, b, s)
                    else:
                        assert np.abs(got - want).max() <= 1, (op, b, s)
    rates = {op: round(v / (total / len(ops)) * 1e6, 1) for op, v in bad.items()}
    print(f"differing pixels per 10^6 against torchvision ({'NEAREST' if interp == TR.NEAREST else 'BILINEAR'}): {rates}")
    assert all(r <= 200 for r in rates.values()), rates             # measured: at most 65 (BILINEAR shears), DESIGN §3.26


def test_erase_rule_is_get_params(monkeypatch):
    """RandomErasing.get_params with its uniforms replaced by the device's s and lr and its randints by umulhi of the device's words
    gives the replay's box when the replay takes torch's float32 exp, and the original image (no erase) where none fits"""
    i = np.arange(400, dtype=np.uint64) * np.uint64(104729)
    for (h, w), scale, ratio in [((224, 224), (0.02, 0.33), (0.3, 3.3)), ((28, 32), (0.02, 0.33), (0.3, 3.3)),
                                 ((8, 8), (0.5, 1.0), (0.1, 10.0)), ((1, 1), (0.02, 0.33), (0.3, 3.3))]:
        s, lr, wt, wl = TR.erase_draws(i, scale, ratio, SEED, 5)
        torch_exp = lambda v: torch.exp(torch.from_numpy(np.asarray(v, np.float32))).numpy()
        got = TR.choose_erase(h, w, s, lr, wt, wl, exp=torch_exp)
        queue, words = [], []
        monkeypatch.setattr(torch.Tensor, "uniform_", lambda self, a, b: self.fill_(float(queue.pop(0))))
        monkeypatch.setattr(torch, "randint", lambda lo, hi, size: torch.tensor([int(RR.umulhi(words.pop(0), hi))]))
        img = torch.zeros(3, h, w)
        for k in range(len(i)):
            queue[:] = [v for a in range(RR.ATTEMPTS) for v in (s[k, a], lr[k, a])]
            words[:] = [wt[k], wl[k]]
            top, left, eh, ew, v = T.RandomErasing.get_params(img, scale=scale, ratio=ratio, value=[0.0])
            if got[4][k] < 0:
                assert (top, left, eh, ew) == (0, 0, h, w) and v is img
            else:
                assert (top, left, eh, ew) == tuple(int(a[k]) for a in got[:4]), (k, h, w)
        monkeypatch.undo()


def test_erase_e_changes_over_a_million_draws():
    """how many of 10^6 images' erase boxes change when E replaces torch's float32 exp (224 x 224, the default scale and ratio)"""
    i = np.arange(1_000_000, dtype=np.uint64)
    s, lr, wt, wl = TR.erase_draws(i, (0.02, 0.33), (0.3, 3.3), SEED, 0)
    torch_exp = lambda v: torch.exp(torch.from_numpy(np.asarray(v, np.float32))).numpy()
    e = np.stack(TR.choose_erase(224, 224, s, lr, wt, wl))
    t = np.stack(TR.choose_erase(224, 224, s, lr, wt, wl, exp=torch_exp))
    changed = int(np.any(e != t, axis=0).sum())
    print(f"{changed} of {len(i)} erase boxes change with E in place of torch's exp")
    assert changed <= 20


def test_draw_statistics():
    """op uniform over 14, bin over 31, sign and the erase decision Bernoulli, each count within 5 sigma over 2 10^5 images"""
    n = 200_000
    op, b, sign, ue = TR.draws(np.arange(n, dtype=np.uint64), SEED, 4)
    for v, k in ((op, 14), (b, 31)):
        counts = np.bincount(v, minlength=k)
        assert counts.size == k and np.all(np.abs(counts - n / k) < 5 * math.sqrt(n * (1 / k) * (1 - 1 / k)))
    for p in (0.5, 0.1):
        c = int((ue < np.float32(p)).sum()) if p != 0.5 else int(sign.sum())
        assert abs(c - n * p) < 5 * math.sqrt(n * p * (1 - p))


def test_trivial_counters_are_their_own():
    """word 1 of a trivial counter, for any index below 2^56 and block 0..6, is in 0xD0000000 .. 0xD6FFFFFF: above every box counter
    (top byte 0xC8 .. 0xCD) and permutation round, bit 30 set where a crop counter's is clear, bit 31 where a dropout counter's is"""
    i = np.array([0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 40 + 17, 2 ** 56 - 1], np.uint64)
    words = np.concatenate([TR.counters(i, k, 0)[1] for k in range(7)]).astype(np.uint64)
    assert (words >= 0xD0000000).all() and (words <= 0xD6FFFFFF).all()
    box = np.concatenate([RR.box_counters(i, k, 0)[1] for k in range(6)]).astype(np.uint64)
    assert box.max() < 0xD0000000
    perm = np.array([A.round_counters(np.zeros(1), r, 0)[1] for r in range(A.ROUNDS)], np.uint64)
    assert perm.max() < 0xD0000000
    crop = A.crop_counters(np.array([0, 2 ** 62 - 1], np.uint64), 0)[1]
    assert ((crop & np.uint64(0x40000000)) == 0).all() and ((words & np.uint64(0x40000000)) != 0).all()
    assert ((words & np.uint64(0x80000000)) != 0).all()
    pairs = {(int(a), int(c)) for k in range(7) for a, c in zip(*TR.counters(i, k, 0)[:2])}
    assert len(pairs) == len(i) * 7


def test_replay_batch_geometry_and_identity():
    """with trivial NONE and no erasing the replay is augment_ref's and resize_ref's batch"""
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (20, 12, 10, 3), dtype=np.uint8)
    x, _, i, _ = TR.batch(img, 4, 8, trivial=TR.NONE, pad=2, flip=1, seed=9, epoch=2, C_out=4)
    assert np.array_equal(x, A.batch(img, 4, 8, pad=2, flip=1, seed=9, epoch=2, C_out=4)[0])
    x, _, i, _ = TR.batch(img, 4, 8, trivial=TR.NONE, crop_size=(8, 8), flip=1, seed=9, epoch=2)
    assert np.array_equal(x, RR.batch(img, 4, 8, RR.TRAIN, 8, 8, flip=1, seed=9, epoch=2)[0])


OK = dict(n=64, H=32, W=32, C=3, first=0, N=8, trivial=2, erase_p=0.25, erase_scale=(0.02, 0.33), erase_ratio=(0.3, 3.3),
          crop_size=None, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3), shuffle=1, pad=4, flip=1, C_out=8, row_pitch=0, image_rows=0, mean=None,
          std=None)
F = "pcnn_augment_trivial_u8_bf16_info: "
REFUSALS = [
    (dict(trivial=3), F + "trivial = 3: 0 \\(none\\), 1 \\(NEAREST\\) or 2 \\(BILINEAR\\) is required"),
    (dict(trivial=-1), "trivial = -1"),
    (dict(C=2, C_out=8), "C = 2: TrivialAugmentWide takes C = 1 or 3"),
    (dict(C=4, C_out=8), "C = 4: TrivialAugmentWide takes C = 1 or 3"),
    (dict(erase_p=1.5), "erase_p = 1.5: a finite 0 <= p <= 1 is required"),
    (dict(erase_p=float("nan")), "erase_p = nan"),
    (dict(erase_p=-0.1), "erase_p = -0.1"),
    (dict(erase_scale=(0.5, 0.2)), "erase scale = \\(0.5, 0.2\\): 0 <= s0 <= s1 <= 1 is required"),
    (dict(erase_scale=(-0.1, 0.2)), "erase scale = \\(-0.1, 0.2\\)"),
    (dict(erase_scale=(0.1, 1.5)), "erase scale = \\(0.1, 1.5\\)"),
    (dict(erase_ratio=(0.0, 3.3)), "erase ratio = \\(0, 3.3\\): r0 <= r1, each within fp32's normal range"),
    (dict(erase_ratio=(3.0, 0.3)), "erase ratio = \\(3, 0.3\\)"),
    (dict(erase_ratio=(0.3, float("inf"))), "erase ratio = \\(0.3, inf\\)"),
    (dict(crop_size=(24, 24)), "pad = 4: a resized batch takes no padding"),
    (dict(n=0), "n = 0, N = 8, H = 32, W = 32: each must be >= 1"),
    (dict(C_out=2), "C_out = 2: C = 3 <= C_out <= 8 is required"),
    (dict(row_pitch=100), "row_pitch = 100: 0 \\(W C_out = 256 rounded up to 8\\)"),
    (dict(image_rows=31), "image_rows = 31: 0 \\(H\\) or >= H = 32 is required"),
    (dict(std=(1.0, 0.0, 1.0)), "std\\[1\\] = 0: a finite std > 0 is required"),
    (dict(pad=0, crop_size=(24, 24), scale=(0.9, 0.5)), "scale = \\(0.9, 0.5\\), ratio = \\(0.75, 1.33333\\): each range must be"),
    (dict(H=300, W=300, pad=0), "the crop is 300 x 300: at most 65536 pixels \\(256 x 256\\) are allowed"),
    (dict(H=512, W=512, pad=0, crop_size=(257, 256)), "the crop is 257 x 256: at most 65536 pixels"),
    (dict(H=256, W=256, C=4, pad=0, trivial=0), "the crop is 256 x 256 x 4: its 262144 bytes, staged in shared memory, must be "
                                                 "<= 227232 \\(227 KB less the kernel's static shared memory\\)"),
    (dict(H=240, W=240, C=4, pad=0, trivial=0, crop_size=(240, 240)), "the crop is 240 x 240 x 4: its 230400 bytes"),
]


@pytest.mark.parametrize("change,msg", REFUSALS)
def test_info_refusals(pkg, change, msg):
    with pytest.raises(pkg.PcnnError, match=msg):
        pkg.augment_trivial_info(**dict(OK, **change))


def test_refusals_in_a_process_without_a_gpu(pkg):
    """the query answers and refuses with the same messages where no GPU is visible"""
    cases = [OK] + [dict(OK, **c) for c, _ in REFUSALS]
    code = ("import json, math, pcnn_loader; pkg = pcnn_loader.load(); out = []\n"
            f"for a in json.loads({json.dumps(json.dumps(cases))}):\n"
            "    try:\n        out.append(pkg.augment_trivial_info(**a)[0])\n"
            "    except pkg.PcnnError as e:\n        out.append(e.msg)\n"
            "print(json.dumps(out))")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = json.loads(subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, check=True).stdout)
    assert out[0] == pkg.augment_trivial_info(**OK)[0]
    for a, msg in zip(cases[1:], out[1:]):
        with pytest.raises(pkg.PcnnError) as e:
            pkg.augment_trivial_info(**a)
        assert msg == e.value.msg


@pytest.mark.parametrize("h,w,C,smem", [(224, 224, 3, 150528), (256, 256, 3, 196608), (28, 32, 1, 896), (5, 7, 3, 112),
                                        (238, 238, 4, 226576)])
def test_info_launch(pkg, h, w, C, smem):
    """one CTA of 512 threads per image with the crop's h w C bytes (rounded up to 16) of dynamic shared memory, which with the
    static part fits the 227 KB an H100 CTA may opt into; the workspace is N h ws_pitch uint16"""
    info = pkg.augment_trivial_info(300, h, w, C, 0, 256, 0 if C == 4 else 1, 0.5 if C == 4 else 0.0, pad=0)[0]
    assert (info["h"], info["w"], info["threads"], info["grid"], info["smem"]) == (h, w, 512, 256, smem)
    assert info["smem"] + info["static_smem"] <= 227 * 1024
    assert info["ws_pitch"] == -(-w * C // 8) * 8 and info["ws_bytes"] == 256 * h * info["ws_pitch"] * 2
    assert info["arg_bytes"] <= 32764


def test_batcher_refuses_before_touching_the_engine(pkg):
    img = np.zeros((16, 8, 8, 3), np.uint8)
    lab = np.zeros(16, np.uint8)
    with pytest.raises(pkg.PcnnError, match="trivial_augment = 'bicubic': None, 'nearest' or 'bilinear' is required"):
        pkg.ImageBatcher(None, img, lab, 4, trivial_augment="bicubic")
    with pytest.raises(pkg.PcnnError, match="trivial_augment = True"):
        pkg.ImageBatcher(None, img, lab, 4, trivial_augment=True)
    for p in (1.5, -0.1, float("nan"), "0.5"):
        with pytest.raises(pkg.PcnnError, match="random_erase = .*: a probability 0 <= p <= 1 is required"):
            pkg.ImageBatcher(None, img, lab, 4, random_erase=p)
    for kw in (dict(trivial_augment="nearest"), dict(random_erase=0.5)):
        for mix in (dict(mixup_alpha=0.2), dict(cutmix_alpha=1.0)):
            with pytest.raises(pkg.PcnnError, match="trivial_augment or random_erase with mixup_alpha or cutmix_alpha > 0"):
                pkg.ImageBatcher(None, img, lab, 4, **kw, **mix)
    with pytest.raises(pkg.PcnnError, match="C = 4: TrivialAugmentWide takes C = 1 or 3"):
        pkg.ImageBatcher(None, np.zeros((16, 8, 8, 4), np.uint8), lab, 4, trivial_augment="bilinear")
    with pytest.raises(pkg.PcnnError, match="erase scale = \\(0.5, 0.2\\)"):
        pkg.ImageBatcher(None, img, lab, 4, random_erase=0.5, erase_scale=(0.5, 0.2))
    with pytest.raises(pkg.PcnnError, match="erase ratio = \\(0, 3.3\\)"):
        pkg.ImageBatcher(None, img, lab, 4, random_erase=0.5, erase_ratio=(0.0, 3.3))
    with pytest.raises(pkg.PcnnError, match="the crop is 300 x 300"):
        pkg.ImageBatcher(None, np.zeros((4, 300, 300, 3), np.uint8), None, 4, trivial_augment="nearest")
