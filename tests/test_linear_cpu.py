"""The fully connected layer and the bf16 softmax cross-entropy without a GPU: the float64 references of linear_ref.py pinned to
torch (functional.linear, cross_entropy, autograd), and pcnn_linear_info over a grid of shapes: every refusal with its message,
the row pitch default and splits that depend on the shape alone."""
import itertools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import linear_ref as LR


@pytest.mark.parametrize("N,P,Q,C,O,act", [(5, 3, 2, 7, 10, 0), (9, 1, 1, 24, 3, 1), (4, 6, 6, 16, 128, 1), (3, 2, 5, 1, 1, 0)])
def test_reference_matches_torch(N, P, Q, C, O, act):
    rng = np.random.default_rng(N * 1000 + O)
    x, w, b = rng.normal(size=(N, P, Q, C)), rng.normal(size=(O, P, Q, C)), rng.normal(size=O)
    xt = torch.tensor(x, requires_grad=True)
    wt = torch.tensor(w, requires_grad=True)
    bt = torch.tensor(b, requires_grad=True)
    pre = F.linear(xt.reshape(N, -1), wt.reshape(O, -1), bt)
    y = torch.sigmoid(pre) if act else pre
    np.testing.assert_allclose(LR.fwd_f64(x, w, b, act), y.detach().numpy(), rtol=1e-13, atol=1e-13)
    dy = rng.normal(size=(N, O))
    y.backward(torch.tensor(dy))
    dpre = dy * (LR.fwd_f64(x, w, b, 1) * (1 - LR.fwd_f64(x, w, b, 1))) if act else dy
    np.testing.assert_allclose(LR.wgrad_f64(x, dpre), wt.grad.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(LR.dgrad_f64(dpre, w), xt.grad.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dpre.sum(axis=0), bt.grad.numpy(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("N,O,scale", [(7, 10, 1 / 7), (33, 1, 1.0), (5, 256, 0.25)])
def test_softmax_ce_reference_matches_torch(N, O, scale):
    rng = np.random.default_rng(O)
    z = rng.normal(0, 3, (N, O))
    lab = rng.integers(0, O, N)
    zt = torch.tensor(z, requires_grad=True)
    loss = F.cross_entropy(zt, torch.tensor(lab), reduction="sum") * scale
    loss.backward()
    g, l, pred = LR.softmax_ce_f64(z, lab, scale)
    np.testing.assert_allclose(l.sum() * scale, loss.item(), rtol=1e-12)
    np.testing.assert_allclose(g, zt.grad.numpy(), rtol=1e-12, atol=1e-15)
    assert np.array_equal(pred, np.argmax(z, axis=1))


def test_softmax_ce_reference_special_rows():
    z = np.array([[1.0, 3.0, 3.0, 0.0], [np.nan, 1.0, 2.0, 0.0], [-np.inf] * 4, [0.0, 1.0, 2.0, 3.0]])
    g, l, pred = LR.softmax_ce_f64(z, np.array([0, 1, 2, 9]), 1.0)
    assert list(pred) == [1, -1, 0, 3]                              # first maximum; NaN row -1; all -Inf: index 0
    assert np.isnan(l[1]) and np.isnan(g[1]).all() and np.isnan(l[3]) and np.isnan(g[3]).all()
    assert np.isfinite(g[0]).all() and np.isfinite(l[0])


def _expected_info(N, P, Q, C, O, row_pitch, image_rows):
    """pcnn_linear_info restated: every split from the shape alone (128 target units, never the SM count)"""
    nch = -(-(Q * C) // 64)
    mt = -(-N // 128)
    steps = P * nch
    fs = max(1, min(-(-128 // mt), steps // 8))
    pairs = (steps + 1) // 2
    ws = min(-(-128 // pairs), mt)
    nb = min(4, steps)
    return dict(row_pitch=row_pitch or (Q * C + 7) // 8 * 8, image_tiles=mt, fwd_steps=steps, fwd_splits=fs, wgrad_pairs=pairs,
                wgrad_splits=ws, dgrad_tiles=mt * -(-steps // nb), dgrad_chunks=nb, npad=(O + 15) // 16 * 16)


def test_info_grid(pkg):
    n = 0
    for N, P, Q, C, O in itertools.product((1, 100, 128, 1024, 4096), (1, 6, 7), (1, 5, 7), (1, 16, 26, 256), (1, 10, 120, 256)):
        if P * Q * C > 1 << 24:
            continue
        for pitch, rows in ((0, 0), ((Q * C + 7) // 8 * 8 + 8, P + 2)):
            got = pkg.linear_info(N, P, Q, C, O, pitch, rows)
            exp = _expected_info(N, P, Q, C, O, pitch, rows)
            assert {k: got[k] for k in exp} == exp, (N, P, Q, C, O, pitch, rows)
            assert 1 <= got["fwd_stages"] <= 8 and 1 <= got["wgrad_stages"] <= 8 and 1 <= got["dgrad_stages"] <= 8
            assert pkg.linear_info(N, P, Q, C, O, pitch, rows) == got
            n += 1
    assert n > 500
    # the benchmark heads
    assert pkg.linear_info(1024, 7, 7, 256, 256)["fwd_splits"] == 16
    assert pkg.linear_info(4096, 1, 1, 2048, 256)["wgrad_splits"] == 8
    assert pkg.linear_info(128, 1, 1, 128, 10)["fwd_splits"] == 1


@pytest.mark.parametrize("args,msg", [
    ((0, 1, 1, 8, 10, 0, 0), r"N, P, Q, C >= 1 and 1 <= O <= 256"),
    ((4, 0, 1, 8, 10, 0, 0), r"N, P, Q, C >= 1 and 1 <= O <= 256"),
    ((4, 1, 0, 8, 10, 0, 0), r"N, P, Q, C >= 1 and 1 <= O <= 256"),
    ((4, 1, 1, 0, 10, 0, 0), r"N, P, Q, C >= 1 and 1 <= O <= 256"),
    ((4, 1, 1, 8, 0, 0, 0), r"N, P, Q, C >= 1 and 1 <= O <= 256"),
    ((4, 1, 1, 8, 257, 0, 0), r"N, P, Q, C >= 1 and 1 <= O <= 256"),
    ((4, 64, 64, 4097, 10, 0, 0), r"at most 2\^24"),
    ((4, 1, 1, 10, 10, 10, 0), r"row pitch 10 must be >= Q\*C = 10 and a multiple of 8.*hidden width.*multiple of 8"),
    ((4, 2, 3, 8, 10, 16, 0), r"row pitch 16 must be >= Q\*C = 24"),
    ((4, 3, 3, 8, 10, 0, 2), r"image pitch of 2 rows is smaller than P = 3"),
])
def test_info_refusals(pkg, args, msg):
    with pytest.raises(pkg.PcnnError, match="pcnn_linear_plan_create: .*" + msg):
        pkg.linear_info(*args)


def test_info_row_pitch_default(pkg):
    for Q, C in ((1, 10), (5, 26), (6, 16), (1, 128), (7, 3)):
        assert pkg.linear_info(8, 2, Q, C, 10)["row_pitch"] == (Q * C + 7) // 8 * 8
