"""GPU tests of the persistent cooperative training kernel (csrc/persist_kernels.cu) and of the multi-GPU step.

Single GPU: the persistent kernel (grid barriers, in-kernel reduction + update) must reproduce the graph path's
parameters: the per-CTA partial gradients are identical, only the fixed summation tree over slots differs, so the bound
is a few ulp per step (rel-L2 <= 2e-6 after 40 steps), and both satisfy the oracle bound of test_fused_gpu.py.
Multi GPU (needs >= 2 visible GPUs, spawned with torch.distributed.run): data-parallel steps over NCCL (graph mode) and
over the in-kernel NVLink exchange (persistent mode) must equal a single-GPU run on the global batch (rel-L2 <= 5e-6)
and leave bit-identical replicas on all ranks.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


@pytest.mark.parametrize("B,steps", [(1, 300), (7, 40), (256, 40), (1024, 3)])
def test_persistent_equals_graph_mode(eng, pkg, golden, B, steps):
    n = 1000
    eng.dataset_upload(pkg.TRAIN_SET, golden["train_u8"][:n], golden["train_labels"][:n])
    out = {}
    for mode in (pkg.MODE_GRAPH, pkg.MODE_PERSISTENT):
        eng.set_step_mode(mode)
        eng.set_params(golden["params_init"])
        eng.err_sum(reset=True)
        l0 = eng.launch_count()
        eng.train_steps(0, B, steps)          # wraps around the 1000-sample split for the larger batches
        eng.sync()
        out[mode] = (eng.get_params(), eng.err_sum(), eng.launch_count() - l0, eng.get_grads())
    eng.set_step_mode(pkg.MODE_AUTO)
    pg, eg, lg, gg = out[pkg.MODE_GRAPH]
    pp, ep, lp, gp = out[pkg.MODE_PERSISTENT]
    assert lp == 1 and lg == 3 * steps                     # one cooperative launch vs three kernels per step
    assert rel_l2(pp, pg) <= 2e-6
    assert rel_l2(gp, gg) <= 1e-5
    assert abs(ep - eg) <= 1e-5 * abs(eg)


def test_persistent_is_default_and_deterministic(eng, pkg, golden):
    n = 1000
    eng.dataset_upload(pkg.TRAIN_SET, golden["train_u8"][:n], golden["train_labels"][:n])
    runs = []
    for _ in range(2):
        eng.set_params(golden["params_init"])
        l0 = eng.launch_count()
        eng.learn(B=64, epochs=2)                        # 16 steps per epoch, ragged tail of 40 samples
        runs.append(eng.get_params())
        assert eng.launch_count() - l0 == 2              # AUTO picks the persistent kernel: one launch per epoch
    assert np.array_equal(runs[0].view(np.uint32), runs[1].view(np.uint32))
    # against the oracle, step by step with the tail batch
    p = golden["params_init"]
    f32 = O.u8_to_f32(golden["train_u8"][:n])
    for _ in range(2):
        for lo in range(0, n, 64):
            hi = min(n, lo + 64)
            g, _ = O.batch_grad(p, f32[lo:hi], golden["train_labels"][lo:hi])
            p = O.apply_update(p, g.astype(np.float32), np.float32(0.1) / np.float32(hi - lo))
    np.testing.assert_allclose(runs[0], p, rtol=2e-5, atol=2e-6)


def _gpu_count():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=30).stdout
        return sum(1 for line in out.splitlines() if line.startswith("GPU "))
    except Exception:
        return 0


def _world():
    """All visible GPUs of the box, at most 8 (the driver's 1-GPU lease skips these cases; gpurun --gpus N runs them)."""
    return min(8, _gpu_count())


@pytest.mark.skipif(_gpu_count() < 2, reason="needs at least 2 GPUs (run with gpurun --gpus 2)")
@pytest.mark.parametrize("batch", [64, 1024])
@pytest.mark.parametrize("mode", ["nccl", "p2p"])
def test_data_parallel_equals_single_gpu(mode, batch):
    """SURVEY.md 8a x4: `world` GPUs x `batch` images against ONE GPU on the global batch (world = 8, batch = 1024 is
    BASELINE config 4: 8 x 1024 vs 1 x 8192), same steps: parameters within rel-L2 1e-6, replicas bit-identical."""
    world = _world()
    port = 29600 + (os.getpid() % 300) + (0 if mode == "nccl" else 301) + (17 if batch == 1024 else 0)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(O.ROOT, "tests", "mgpu_worker.py"), "--mode", mode, "--batch", str(batch),
           "--steps", "20" if batch == 64 else "4"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "MGPU_OK" in r.stdout, r.stdout[-3000:]
    log_dir = os.environ.get("PCNN_MGPU_LOG_DIR")
    if log_dir:      # optional: keep the workers' parity lines as a log
        with open(os.path.join(log_dir, f"mgpu_parity_n{world}.log"), "a") as f:
            f.write("".join(ln + "\n" for ln in r.stdout.splitlines() if "mode=" in ln or "MGPU" in ln))
