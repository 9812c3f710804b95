"""Dropout and stochastic depth without a GPU: the numpy Philox4x32-10 of dropout_ref.py against the Random123 known-answer vectors,
the keep rate and independence of its masks, and pcnn_dropout_bf16_info (T, scale, path and launch), including in a process that
sees no GPU, with every refusal."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import dropout_ref as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Random123's kat_vectors for philox4x32_10: (counter, key) -> output
KAT = [((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff, 0xffffffff, 0xffffffff, 0xffffffff), (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(w) for w in D.philox4x32_10(ctr, key)) == want


def test_philox_vectorised_matches_scalar():
    """an array of counters gives, element by element, what each counter gives alone; the draw of index i is word i & 3"""
    q = np.array([0, 1, 7, 0xFFFFFFFF], np.uint64)
    batch = D.philox4x32_10((q, 0, 5, 0), (11, 0))
    for k, c in enumerate(q):
        assert np.array_equal(batch[k], D.philox4x32_10((int(c), 0, 5, 0), (11, 0)))
    i = np.arange(16, dtype=np.uint64)
    assert np.array_equal(D.draws(i, 11, 5), D.philox4x32_10((np.arange(4, dtype=np.uint64), 0, 5, 0), (11, 0)).reshape(-1))
    # the upper words of the counter and the key are used: index 2^34 and call / seed 2^32 move the draws
    assert D.draws(np.array([1 << 34], np.uint64), 11, 5)[0] != D.draws(np.array([0], np.uint64), 11, 5)[0]
    assert not np.array_equal(D.draws(i, 11, 5 + (1 << 32)), D.draws(i, 11, 5))
    assert not np.array_equal(D.draws(i, 11 + (1 << 32), 5), D.draws(i, 11, 5))


def test_threshold_rule():
    assert D.threshold(0.0) == (0, np.float32(1.0))
    assert D.threshold(0.5) == (1 << 31, np.float32(2.0))
    assert D.threshold(0.2) == (858993459, np.float32(1.25))          # 0.2 * 2^32 = 858993459.2
    assert D.threshold(0.1)[1] == np.float32(1.0 / 0.9)
    assert D.threshold(1 - 2.0 ** -34)[0] == 0xFFFFFFFF             # nearest is 2^32: the largest uint32
    assert D.threshold(2.0 ** -33)[0] == 0                           # 1/2: ties to even
    assert D.threshold(3 * 2.0 ** -33)[0] == 2


@pytest.mark.parametrize("p", [0.1, 0.2, 0.5])
def test_keep_rate(p):
    """over 2^22 draws the kept fraction is within 5 sigma of 1 - p"""
    n = 1 << 22
    kept = D.keep(1 << 10, n >> 10, p, seed=12345, call=1)
    sigma = np.sqrt(p * (1 - p) / n)
    assert abs(kept.mean() - (1 - p)) < 5 * sigma, (kept.mean(), 1 - p)


def test_masks_independent():
    """masks of different calls and seeds agree at the rate of independent masks, (1 - p)^2 + p^2; per-sample masks are whole rows"""
    p, n = 0.5, 1 << 20
    base = D.keep(1024, n >> 10, p, seed=7, call=1)
    sigma = np.sqrt(0.25 / n)
    for other in (D.keep(1024, n >> 10, p, seed=7, call=2), D.keep(1024, n >> 10, p, seed=8, call=1),
                  D.keep(1024, n >> 10, p, seed=7 + (1 << 32), call=1)):
        assert abs((base == other).mean() - 0.5) < 5 * sigma
    rows = D.keep(4096, 3, 0.2, seed=7, call=1, per_sample=True)
    assert (rows == rows[:, :1]).all()
    assert abs(rows[:, 0].mean() - 0.8) < 5 * np.sqrt(0.16 / 4096)


def test_values():
    x = np.array([[1.5, -2.0, np.nan, np.inf, -0.0, 1e-40, 3.0, -1.0]], np.float32)
    kept = np.array([[True, False, False, False, False, True, True, False]])
    y = D.values(x, kept, np.float32(1.25))
    assert y[0, 0] == 1.875 and np.isnan(y[0, 2]) and np.isnan(y[0, 3])
    assert y[0, 1] == 0 and np.signbit(y[0, 1]) and np.signbit(y[0, 7])          # a dropped -x gives -0
    r = np.full_like(x, 2.0)
    yr = D.values(x, kept, np.float32(1.25), r)
    assert yr[0, 1] == 2.0 and yr[0, 0] == D.bf16(np.float32(2.0) + np.float32(1.875))


INFO = [  # N, row_elems, row_pitch, p, per_sample, vec
    (128, 56 * 56 * 64, 0, 0.2, 0, 8), (128, 7 * 7 * 1280, 0, 0.5, 1, 8), (128, 12, 16, 0.2, 0, 1), (128, 1280, 1280, 0.1, 0, 8),
    (1, 3, 0, 0.9, 0, 1), (7, 24, 25, 0.3, 1, 1), (5, 8, 0, 0.0, 0, 8)]


@pytest.mark.parametrize("N,E,pitch,p,ps,vec", INFO)
def test_info(pkg, N, E, pitch, p, ps, vec):
    got = pkg.dropout_info(N, E, pitch, p, ps)
    T, scale = D.threshold(p)
    assert got["T"] == T and got["scale_bits"] == int(scale.view(np.uint32)) and got["vec"] == vec
    vectors = N * E // vec
    assert got["grid"] == min(1056, -(-vectors // 256))
    assert got["per_thread"] == -(-vectors // (got["grid"] * 256)) * vec


def test_info_independent_of_the_device(pkg):
    """pcnn_dropout_bf16_info takes no context: a process that sees no GPU at all gets the same answers"""
    cases = [(c[0], c[1], c[2], c[3], c[4]) for c in INFO]
    code = ("import json, pcnn_loader; pkg = pcnn_loader.load(); "
            f"print(json.dumps([pkg.dropout_info(*c) for c in {cases!r}]))")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, check=True).stdout
    assert json.loads(out) == [pkg.dropout_info(*c) for c in cases]


REFUSALS = [  # args of dropout_info (N, row_elems, row_pitch, p, per_sample), words of the message
    ((0, 8, 0, 0.1, 0), "pcnn_dropout_bf16_info: N = 0, row_elems = 8: each must be >= 1"),
    ((4, 0, 0, 0.1, 0), "row_elems = 0: each must be >= 1"),
    ((4, -3, 0, 0.1, 0), "each must be >= 1"),
    ((4, 16, 8, 0.1, 0), "row_pitch = 8: 0 \\(dense\\) or >= row_elems = 16 is required"),
    ((4, 16, -1, 0.1, 0), "row_pitch = -1"),
    ((4, 16, 0, 1.0, 0), "p = 1: a finite p with 0 <= p < 1 is required"),
    ((4, 16, 0, -0.1, 0), "p = -0.1: a finite p"),
    ((4, 16, 0, float("nan"), 0), "p = nan: a finite p"),
    ((4, 16, 0, float("inf"), 0), "p = inf: a finite p"),
    ((4, 16, 0, 0.1, 2), "per_sample = 2: 0 \\(element\\) or 1 \\(per sample\\) is required"),
    ((4, 16, 0, 0.1, -1), "per_sample = -1"),
]


@pytest.mark.parametrize("args,msg", REFUSALS)
def test_info_refusals(pkg, args, msg):
    with pytest.raises(pkg.PcnnError, match=msg):
        pkg.dropout_info(*args)


def test_layer_refuses_before_touching_the_engine(pkg):
    with pytest.raises(pkg.PcnnError, match="p = 1.5"):
        pkg.DropoutLayer(None, 4, 16, 1.5, seed=1)
    layer = pkg.DropoutLayer(None, 4, 16, 0.2, seed=1)
    assert layer.call == 0
    with pytest.raises(pkg.PcnnError, match="no training forward"):
        layer.backward(None, None)
