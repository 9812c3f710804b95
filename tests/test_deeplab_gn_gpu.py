"""DeepLabGN (tests/groupnorm_nets.py) trained on the device at a batch of 4 with segment_nets' harness: in each of the first five
steps every group normalization is checked on its own operands (y, dr and dx bit for bit against groupnorm_ref's replays on the
layer's saved statistics and dstat, the statistics, dgamma, dbeta and dstat within their float64 bounds); a fresh run reproduces
the parameters after five steps bit for bit; and the test mIoU after training is within 0.05 of the float32 replica's
(scripts/deeplab_gn_replica.py)."""
import numpy as np
import pytest

import bnact_ref as BA
import groupnorm_nets
import groupnorm_ref as GR
from example_nets import host
import segment_nets

pytestmark = pytest.mark.gpu

REPLICA_MIOU = 0.6542   # scripts/deeplab_gn_replica.py


def _bits(buf, shape):
    return host(buf).reshape(shape)


def check_norm(pkg, L, x, r, y, dy, dy2, dx, dr):
    N, H, W, C = L.shape
    G, shape = L.groups, (N, H * W, C)
    xb, yb, dyb = _bits(x, shape), _bits(y, shape), _bits(dy, shape)
    rb = None if r is None else _bits(r, shape)
    dy2b = None if dy2 is None else _bits(dy2, shape)
    gamma, beta = L.gamma.to_host(), L.beta.to_host()
    mean, rstd = L.save_mean.to_host().reshape(N, G), L.save_rstd.to_host().reshape(N, G)
    assert np.array_equal(yb, GR.fwd_bits(pkg, xb, gamma, beta, mean, rstd, rb, L.act)), "y"
    GR.check_stats(pkg, xb, G, mean, rstd, L.eps, L.info["n_acc_group"])
    g = GR.grad_bits(pkg, xb, gamma, beta, mean, rstd, dyb, dy2b, rb if L.act in BA.CODES else None, L.act, yb)
    if dr is not None:
        assert np.array_equal(_bits(dr, shape), g), "dr"
    ds = L.dstat.to_host()
    assert np.array_equal(_bits(dx, shape), GR.dx_bits(pkg, xb, g, gamma, mean, rstd, ds)), "dx"
    return GR.check_sums(pkg, xb, g, gamma, mean, rstd, G, L.dgamma.to_host(), L.dbeta.to_host(), ds, L.info)


def test_deeplab_gn_trains(eng, pkg, golden):
    """five checked steps, a bit-identical fresh run, and the trained test mIoU near the float32 replica's (and above twice the
    all-background score)"""
    checked, worst = [], {}

    def check_step(net, it, x, labels, masks):
        net.forward(x, labels, masks)
        net.backward()
        eng.sync()
        for args in net.norms():
            for k, v in check_norm(pkg, *args).items():
                worst[k] = max(worst.get(k, 0.0), v)
        checked.append(it)

    losses, miou, bg, _ = segment_nets.train_segmenter(eng, pkg, golden, groupnorm_nets.DeepLabGN, check_step)
    print(f"DeepLabGN: epoch losses {losses}, test mIoU {miou:.4f} (replica {REPLICA_MIOU:.4f}), all-background mIoU {bg:.4f}; "
          f"worst ratios to the sum bounds {worst}")
    assert checked == [0, 1, 2, 3, 4]
    assert losses[-1] < losses[0]
    assert abs(miou - REPLICA_MIOU) <= 0.05 and miou > 2 * bg
    _, again, _, _ = segment_nets.train_segmenter(eng, pkg, golden, groupnorm_nets.DeepLabGN)
    assert again == miou
