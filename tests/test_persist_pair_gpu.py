"""GPU tests of the two-image CTA of the persistent kernel (csrc/persist_kernels.cu, IPC = 2): when the batch outnumbers the
SMs, one 448-thread CTA per SM trains two images and adds their gradients in shared memory before pushing them.  Only the
order of fp32 sums differs from the single-image CTAs, so the bounds are those of test_persist_gpu.py.  An H100 80GB HBM3
keeps 120 such CTAs co-resident in clusters of 4 (batches up to 240) and 128 in clusters of 2 (a batch of 256)."""
import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def _upload(eng, pkg, golden, n=1000):
    eng.dataset_upload(pkg.TRAIN_SET, golden["train_u8"][:n], golden["train_labels"][:n])


@pytest.mark.parametrize("B,grid,cluster", [(200, 100, 4), (256, 128, 2)])
def test_batch_runs_two_images_per_cta(eng, pkg, golden, B, grid, cluster):
    _upload(eng, pkg, golden)
    eng.set_step_mode(pkg.MODE_PERSISTENT)
    eng.set_params(golden["params_init"])
    eng.train_steps(0, B, 2)
    eng.sync()
    info = eng.persist_info()
    eng.set_step_mode(pkg.MODE_AUTO)
    assert info["images_per_cta"] == 2, info
    assert info["grid"] == grid and info["cluster"] == cluster, info


def test_small_batch_keeps_one_image_per_cta(eng, pkg, golden):
    _upload(eng, pkg, golden)
    eng.set_step_mode(pkg.MODE_PERSISTENT)
    eng.set_params(golden["params_init"])
    eng.train_steps(0, 64, 2)
    eng.sync()
    info = eng.persist_info()
    eng.set_step_mode(pkg.MODE_AUTO)
    assert info["images_per_cta"] == 1 and info["grid"] == 64, info


@pytest.mark.parametrize("B", [153, 199, 255])
def test_odd_batch_equals_graph_mode(eng, pkg, golden, B):
    """The last CTA with an image has only image 2c; its half 1 contributes zeros."""
    _upload(eng, pkg, golden)
    steps = 40
    out = {}
    for mode in (pkg.MODE_GRAPH, pkg.MODE_PERSISTENT):
        eng.set_step_mode(mode)
        eng.set_params(golden["params_init"])
        eng.err_sum(reset=True)
        eng.train_steps(0, B, steps)
        eng.sync()
        out[mode] = (eng.get_params(), eng.err_sum(), eng.get_grads())
    info = eng.persist_info()
    eng.set_step_mode(pkg.MODE_AUTO)
    assert info["images_per_cta"] == 2, info
    pg, eg, gg = out[pkg.MODE_GRAPH]
    pp, ep, gp = out[pkg.MODE_PERSISTENT]
    assert rel_l2(pp, pg) <= 2e-6
    assert rel_l2(gp, gg) <= 1e-5
    assert abs(ep - eg) <= 1e-5 * abs(eg)


def test_pair_runs_are_bit_identical(eng, pkg, golden):
    _upload(eng, pkg, golden)
    eng.set_step_mode(pkg.MODE_PERSISTENT)
    runs = []
    for _ in range(2):
        eng.set_params(golden["params_init"])
        eng.err_sum(reset=True)
        eng.train_steps(0, 200, 30)
        eng.sync()
        runs.append((eng.get_params(), eng.get_grads(), eng.err_sum()))
    eng.set_step_mode(pkg.MODE_AUTO)
    assert np.array_equal(runs[0][0].view(np.uint32), runs[1][0].view(np.uint32))
    assert np.array_equal(runs[0][1].view(np.uint32), runs[1][1].view(np.uint32))
    assert runs[0][2] == runs[1][2]


def test_learn_192_with_ragged_tail_matches_oracle(eng, pkg, golden):
    n = 1000
    _upload(eng, pkg, golden, n)
    eng.set_params(golden["params_init"])
    l0 = eng.launch_count()
    eng.learn(B=192, epochs=1)                         # five batches of 192, then a tail of 40 in the same 96 two-image CTAs
    got = eng.get_params()
    assert eng.launch_count() - l0 == 1
    assert eng.persist_info()["images_per_cta"] == 2
    p = golden["params_init"]
    f32 = O.u8_to_f32(golden["train_u8"][:n])
    for lo in range(0, n, 192):
        hi = min(n, lo + 192)
        g, _ = O.batch_grad(p, f32[lo:hi], golden["train_labels"][lo:hi])
        p = O.apply_update(p, g.astype(np.float32), np.float32(0.1) / np.float32(hi - lo))
    np.testing.assert_allclose(got, p, rtol=2e-5, atol=2e-6)
