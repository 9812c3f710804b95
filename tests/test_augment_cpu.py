"""The input pipeline without a GPU: the numpy replay of augment_ref.py (the permutation is a bijection that moves between epochs,
its first position is uniform, the crop offsets and flips are uniform, and no counter it draws at is one dropout can draw at), and
pcnn_augment_u8_bf16_info (layout, permutation width, launch and the value table against torch), including in a process that
sees no GPU, with every refusal."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import augment_ref as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEEDS = (0, 0x0123456789ABCDEF, (1 << 64) - 1)


@pytest.mark.parametrize("n", [1, 2, 3, 5, 255, 256, 1000, 1024, 60000, (1 << 20) + 7])
def test_permutation_is_a_bijection(n):
    """pi is a permutation of [0, n) for 3 seeds x 3 epochs, and consecutive epochs differ for n >= 4"""
    e = np.arange(n, dtype=np.uint64)
    walks = []
    for seed in SEEDS:
        perms = []
        for epoch in (0, 1, (1 << 40) + 3):
            p, w = A.permute(e, n, seed, epoch, walks=True)
            assert np.array_equal(np.sort(p), e), (n, seed, epoch)
            perms.append(p)
            walks.append(w)
        if n >= 4:
            assert not np.array_equal(perms[0], perms[1]) and not np.array_equal(perms[1], perms[2]), (n, seed)
    w = np.concatenate(walks)
    assert w.max() < 4 * 2 ** (2 * A.half_width(n)) and w.mean() < 4.0
    print(f"n = {n}: b = {A.half_width(n)}, applications of the network per position: mean {w.mean():.3f}, longest {w.max()}")


def test_permutation_depends_on_n_seed_and_epoch_alone():
    """a prefix of positions permutes as the whole epoch does (no dependence on N or first), and pi(e) depends on the seed"""
    n = 1000
    full = A.permute(np.arange(n, dtype=np.uint64), n, 5, 2)
    assert np.array_equal(A.permute(np.arange(300, 428, dtype=np.uint64), n, 5, 2), full[300:428])
    assert not np.array_equal(A.permute(np.arange(n, dtype=np.uint64), n, 6, 2), full)


@pytest.mark.parametrize("n", [2, 3, 4, 5, 6, 7, 10, 17, 33])
def test_first_position_uniform(n):
    """over 40000 epochs pi(0) takes each of the n values within 5 sigma of 1 / n"""
    E = 40000
    f = A.permute(np.zeros(E, np.uint64), n, 7, np.arange(E, dtype=np.uint64)).astype(np.int64)
    count = np.bincount(f, minlength=n)
    sigma = np.sqrt(E * (1 / n) * (1 - 1 / n))
    assert np.abs(count - E / n).max() < 5 * sigma, count


@pytest.mark.parametrize("pad", [1, 2, 4, 64])
def test_offsets_and_flips_uniform(pad):
    """over 2^20 images oy and ox take each value of [0, 2 pad] within 5 sigma, and the flip rate is 1/2 within 5 sigma"""
    m = 1 << 20
    oy, ox, fl = A.draws(np.arange(m, dtype=np.uint64), pad, 1, 0x0123456789ABCDEF, 3)
    k = 2 * pad + 1
    sigma = np.sqrt(m * (1 / k) * (1 - 1 / k))
    for o in (oy, ox):
        assert o.min() >= 0 and o.max() <= 2 * pad
        assert np.abs(np.bincount(o, minlength=k) - m / k).max() < 5 * sigma
    assert abs(fl.mean() - 0.5) < 5 * np.sqrt(0.25 / m)
    assert not A.draws(np.arange(16, dtype=np.uint64), pad, 0, 1, 3)[2].any()      # flip 0: never mirrored


def test_counters_never_dropouts():
    """every counter the pipeline draws at has bit 31 of word 1 set; a dropout counter's word 1 is the high word of an element
    index below 2^62 (N, row_elems < 2^31), so it never is.  The permutation's rounds also set bit 30, which no crop counter
    (i < 2^62) does."""
    i = np.array([0, 1, 59999, (1 << 32) + 5, (1 << 62) - 1], np.uint64)
    crop = A.crop_counters(i, (1 << 63) + 9)
    assert np.all(crop[1] >> np.uint64(31) == 1) and np.all((crop[1] >> np.uint64(30)) & np.uint64(1) == 0)
    for r in range(A.ROUNDS):
        rnd = A.round_counters(np.arange(16, dtype=np.uint64), r, 12)
        assert rnd[1] >> 30 == 3 and rnd[1] & 0x3FFFFFFF == r
    max_dropout_index = (2 ** 31 - 1) * (2 ** 31 - 1) + 2 ** 31 - 2
    assert (max_dropout_index >> 2) >> 32 < 1 << 30
    # the same seed and epoch as a dropout call: different words at the same low counter
    import dropout_ref as D
    assert not np.array_equal(A.draws(np.arange(64, dtype=np.uint64), 4, 1, 7, 1)[0],
                              (D.draws(np.arange(64, dtype=np.uint64), 7, 1).astype(np.uint64) * 9) >> 32)


STATS = [(None, None, 1), (None, None, 3), ((0.4914, 0.4822, 0.4465), (0.2470, 0.2435, 0.2616), 3),
         ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225), 3), ((-0.75, -3.0), (1.0, 1.0), 2), ((0.5,) * 4, (1e-3,) * 4, 4)]


@pytest.mark.parametrize("mean,std,C", STATS, ids=["01-C1", "01-C3", "cifar", "imagenet", "negative-mean", "std-1e-3"])
def test_table_matches_torch(pkg, mean, std, C):
    """the host's table equals torch CPU float32 arange(256).div(255).sub(m).div(s).to(bfloat16), bit for bit"""
    _, lut = pkg.augment_info(64, 8, 8, C, 0, 8, 1, 2, 1, 8, 0, 0, mean, std)
    m = torch.zeros(C) if mean is None else torch.tensor(mean, dtype=torch.float32)
    s = torch.ones(C) if std is None else torch.tensor(std, dtype=torch.float32)
    want = torch.arange(256).float()[None, :].div(255).sub(m[:, None]).div(s[:, None]).to(torch.bfloat16)
    assert np.array_equal(lut, want.view(torch.int16).numpy().view(np.uint16))
    assert np.array_equal(lut, A.table(C, mean, std))
    if mean is None:            # the bits the example networks' mnist_device builds
        assert np.array_equal(lut[0], pkg.f32_to_bf16_bits(np.arange(256, dtype=np.float32) / 255.0))


INFO = [  # n, H, W, C, first, N, shuffle, pad, flip, C_out, row_pitch, image_rows -> row_pitch, image_rows, b, vec, rows_per_cta
    ((1024, 28, 28, 1, 0, 128, 1, 2, 0, 1, 32, 28), (32, 28, 5, 1, 28)),
    ((50000, 32, 32, 3, 512, 512, 1, 4, 1, 3, 0, 0), (96, 32, 8, 8, 32)),
    ((50000, 32, 32, 3, 0, 512, 1, 4, 1, 8, 0, 0), (256, 32, 8, 8, 32)),
    ((2048, 224, 224, 3, 256, 256, 1, 4, 1, 8, 0, 0), (1792, 224, 6, 8, 5)),
    ((100, 27, 31, 1, 3, 7, 0, 3, 1, 1, 40, 30), (40, 30, 4, 1, 27)),
    ((1, 5, 7, 4, 0, 1, 1, 9, 1, 4, 0, 0), (32, 5, 0, 1, 5)),
]


@pytest.mark.parametrize("args,want", INFO)
def test_info(pkg, args, want):
    info, lut = pkg.augment_info(*args)
    assert (info["row_pitch"], info["image_rows"], info["b"], info["vec"], info["rows_per_cta"]) == want
    n, H, W, C, first, N, *_ = args
    assert info["b"] == A.half_width(n) and info["threads"] == 256
    assert info["row_blocks"] == -(-H // info["rows_per_cta"]) and info["grid"] == N * info["row_blocks"]
    assert lut.shape == (C, 256)


def test_info_independent_of_the_device(pkg):
    """pcnn_augment_u8_bf16_info takes no context: a process that sees no GPU at all gets the same answers"""
    cases = [list(c[0]) for c in INFO]
    code = ("import json, pcnn_loader; pkg = pcnn_loader.load(); "
            f"print(json.dumps([[pkg.augment_info(*c)[0], pkg.augment_info(*c)[1].tolist()] for c in {cases!r}]))")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, check=True).stdout
    assert json.loads(out) == [[pkg.augment_info(*c)[0], pkg.augment_info(*c)[1].tolist()] for c in cases]


OK = dict(n=64, H=8, W=8, C=3, first=0, N=8, shuffle=1, pad=2, flip=1, C_out=8, row_pitch=0, image_rows=0, mean=None, std=None)
REFUSALS = [  # changes to OK, words of the message
    (dict(n=0, N=1), "pcnn_augment_u8_bf16_info: n = 0, N = 1, H = 8, W = 8: each must be >= 1"),
    (dict(N=0), "N = 0, H = 8, W = 8: each must be >= 1"),
    (dict(H=0), "H = 0, W = 8: each must be >= 1"),
    (dict(W=-1), "W = -1: each must be >= 1"),
    (dict(first=-1), "first = -1, N = 8: 0 <= first and first \\+ N <= n = 64 are required"),
    (dict(first=57), "first = 57, N = 8: 0 <= first"),
    (dict(N=65), "first = 0, N = 65: 0 <= first"),
    (dict(C=0), "C = 0: 1 <= C <= 4 is required"),
    (dict(C=5), "C = 5: 1 <= C <= 4 is required"),
    (dict(C_out=2), "C_out = 2: C = 3 <= C_out <= 8 is required"),
    (dict(C_out=9), "C_out = 9: C = 3 <= C_out <= 8 is required"),
    (dict(pad=-1), "pad = -1: 0 <= pad <= 64 is required"),
    (dict(pad=65), "pad = 65: 0 <= pad <= 64 is required"),
    (dict(shuffle=2), "shuffle = 2, flip = 1: each must be 0 or 1"),
    (dict(flip=-1), "shuffle = 1, flip = -1: each must be 0 or 1"),
    (dict(H=1 << 16, W=1 << 14, C=2, N=1, first=0), "H W C = 2147483648: one image must fit the 32-bit range"),
    (dict(n=1 << 41, H=1 << 12, W=1 << 10, C=1), "the dataset must be below 2\\^62 bytes"),
    (dict(row_pitch=60), "row_pitch = 60: 0 \\(W C_out = 64 rounded up to 8\\) or a multiple of 8 >= W C_out is required"),
    (dict(row_pitch=68), "row_pitch = 68: 0 \\(W C_out = 64"),
    (dict(row_pitch=-8), "row_pitch = -8"),
    (dict(image_rows=7), "image_rows = 7: 0 \\(H\\) or >= H = 8 is required"),
    (dict(image_rows=-1), "image_rows = -1"),
    (dict(row_pitch=1 << 30, image_rows=1 << 30), "N image_rows row_pitch = 8 x 1073741824 x 1073741824: x must be below 2\\^62 bytes"),
    (dict(mean=(0.0, float("nan"), 0.0)), "mean\\[1\\] = nan: a finite mean is required"),
    (dict(mean=(0.0, 0.0, float("inf"))), "mean\\[2\\] = inf: a finite mean"),
    (dict(std=(1.0, 0.0, 1.0)), "std\\[1\\] = 0: a finite std > 0 is required"),
    (dict(std=(-1.0, 1.0, 1.0)), "std\\[0\\] = -1: a finite std > 0"),
    (dict(std=(1.0, 1.0, float("inf"))), "std\\[2\\] = inf: a finite std > 0"),
    (dict(std=(1.0, float("nan"), 1.0)), "std\\[1\\] = nan: a finite std > 0"),
]


@pytest.mark.parametrize("change,msg", REFUSALS)
def test_info_refusals(pkg, change, msg):
    a = dict(OK, **change)
    with pytest.raises(pkg.PcnnError, match=msg):
        pkg.augment_info(**a)


def test_refusals_in_a_process_without_a_gpu(pkg):
    """the query refuses with the same messages where no GPU is visible"""
    cases = [dict(OK, **c) for c, _ in REFUSALS if all(isinstance(v, int) for v in c.values())]
    code = ("import json, pcnn_loader; pkg = pcnn_loader.load(); out = []\n"
            f"for a in {cases!r}:\n"
            "    try:\n        pkg.augment_info(**a); out.append(None)\n"
            "    except pkg.PcnnError as e:\n        out.append(e.msg)\n"
            "print(json.dumps(out))")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = json.loads(subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, check=True).stdout)
    for a, msg in zip(cases, out):
        with pytest.raises(pkg.PcnnError) as e:
            pkg.augment_info(**a)
        assert msg == e.value.msg


def test_batcher_refuses_before_touching_the_engine(pkg):
    with pytest.raises(pkg.PcnnError, match="pad = 65"):
        pkg.ImageBatcher(None, np.zeros((16, 8, 8, 3), np.uint8), None, 4, pad=65)
    with pytest.raises(pkg.PcnnError, match="uint8"):
        pkg.ImageBatcher(None, np.zeros((16, 8, 8, 3), np.float32), None, 4)
    with pytest.raises(pkg.PcnnError, match="mean has 2 values for C = 3"):
        pkg.ImageBatcher(None, np.zeros((16, 8, 8, 3), np.uint8), None, 4, mean=(0.5, 0.5))
    with pytest.raises(pkg.PcnnError, match="first = 0, N = 17"):
        pkg.ImageBatcher(None, np.zeros((16, 8, 8), np.uint8), None, 17)
