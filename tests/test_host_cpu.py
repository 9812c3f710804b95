"""CPU tests (no GPU) of the host-side logic and of the C-ABI library as a loadable object.  No compute entry point is
called here: without a GPU pcnn_create must fail loudly (no CPU fallback)."""
import ctypes as C
import math
import os
import struct

import numpy as np
import pytest

import oracle_lib as O


def test_library_exports_every_declared_symbol(pkg):
    L = pkg.lib()
    names = pkg.declared_symbols()
    assert len(names) >= 60 and "pcnn_conv_tc_plan_info" in names
    for n in names:
        assert hasattr(L, n), f"libpcnn.so does not export {n} declared in include/pcnn.h"
    assert L.pcnn_version() == 200


def test_sass_is_sm90a_only(pkg):
    import subprocess
    out = subprocess.run(["cuobjdump", "-lelf", pkg.LIB_PATH], capture_output=True, text=True).stdout
    archs = {tok for line in out.splitlines() for tok in line.replace(".", " ").split() if tok.startswith("sm_")}
    assert archs == {"sm_90a"}, archs


def test_init_params_reference_replays_glibc_rand(pkg, golden):
    p = pkg.init_params_reference()
    assert np.array_equal(p.view(np.uint32), golden["params_init"].view(np.uint32))   # the reference's constructor output
    assert np.array_equal(p.view(np.uint32), O.init_params().view(np.uint32))          # the real rand() after srand(1)


def test_create_without_gpu_fails_loudly(pkg):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        pytest.skip("a GPU is present")
    with pytest.raises(pkg.PcnnError) as ei:
        pkg.Engine(0)
    assert ei.value.code == -6 and "no CPU fallback" in str(ei.value)


def test_null_and_bad_arguments_are_rejected_without_a_context(pkg):
    L = pkg.lib()
    assert L.pcnn_sync(None) == -1
    assert L.pcnn_fp_c1(None, None, None, None, None, 1) == -1
    assert L.pcnn_train_step(None, 0, 1) == -1
    assert L.pcnn_init_params_reference(None) == -1
    assert b"NULL" in L.pcnn_last_error_string()
    assert L.pcnn_destroy(None) == 0


def _write_idx(tmp, images, labels, img_magic=2051, lab_magic=2049, lab_count=None, dims=(28, 28)):
    ip, lp = os.path.join(tmp, "img.idx"), os.path.join(tmp, "lab.idx")
    with open(ip, "wb") as f:
        f.write(struct.pack(">IIII", img_magic, len(images), dims[0], dims[1]))
        f.write(images.tobytes())
    with open(lp, "wb") as f:
        f.write(struct.pack(">II", lab_magic, len(labels) if lab_count is None else lab_count))
        f.write(labels.tobytes())
    return ip, lp


def test_mnist_loader_return_codes_follow_mnist_h(pkg, golden, tmp_path):
    tmp = str(tmp_path)
    imgs, labs = golden["train_u8"][:32], golden["train_labels"][:32]
    ip, lp = _write_idx(tmp, imgs, labs)
    rc, a, b = pkg.mnist_load_u8(ip, lp)
    assert rc == 0 and np.array_equal(a, imgs) and np.array_equal(b, labs)
    assert pkg.mnist_load_u8(os.path.join(tmp, "nope"), lp)[0] == -1            # mnist.h:95-98
    assert pkg.mnist_load_u8(*_write_idx(tmp, imgs, labs, img_magic=1234))[0] == -2   # mnist.h:100-104
    assert pkg.mnist_load_u8(*_write_idx(tmp, imgs, labs, lab_magic=1234))[0] == -3   # mnist.h:106-110
    assert pkg.mnist_load_u8(*_write_idx(tmp, imgs, labs, lab_count=31))[0] == -4     # mnist.h:118-121
    assert pkg.mnist_load_u8(*_write_idx(tmp, imgs, labs, dims=(28, 27)))[0] == -2    # mnist.h:128-131


def test_mnist_loader_reads_the_real_idx_files(pkg, golden):
    d = O.REF_DATA
    if not os.path.exists(os.path.join(d, "t10k-images.idx3-ubyte")):
        pytest.skip("full MNIST not staged under oracle/_ref/data")
    rc, a, b = pkg.mnist_load_u8(os.path.join(d, "t10k-images.idx3-ubyte"), os.path.join(d, "t10k-labels.idx1-ubyte"))
    assert rc == 0 and a.shape == (10000, 784)
    assert np.array_equal(a[:256], golden["test_u8"]) and np.array_equal(b[:256], golden["test_labels"])


def test_sharding_covers_the_global_batch_exactly(pkg):
    from parallel_cnn_b200 import sharding as S
    n = 60000
    for B, world in [(1024, 8), (256, 2), (1000, 4), (1, 1), (7, 3)]:
        cursor, seen, steps = 0, 0, 0
        while True:
            ranges = [S.shard(cursor, B, r, world, n) for r in range(world)]
            got = sum(c for _, c in ranges)
            assert got == S.effective_global_batch(cursor, B, world, n)
            # contiguous, non-overlapping, in rank order
            pos = cursor
            for base, cnt in ranges:
                if cnt:
                    assert base == pos
                    pos += cnt
            seen += got
            steps += 1
            cursor = S.next_cursor(cursor, B, world, n)
            if cursor == 0:
                break
        assert seen == n and steps == S.steps_per_epoch(n, B, world)


# --------------------------------------------------------------------------- world_size-2 gloo test of the N > 1 path
def _dp_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import pcnn_loader
    pcnn_loader.load()
    from parallel_cnn_b200 import sharding as S
    d = np.load(os.path.join(O.GOLDEN, "mnist_subset.npz"))
    B, n = 16, 80                                   # 80 samples, global batch 32 -> 3 steps, the last one ragged (16 + 0)
    p = O.init_params()
    cursor = 0
    for _ in range(S.steps_per_epoch(n, B, world)):
        base, cnt = S.shard(cursor, B, rank, world, n)
        if cnt:
            g, es = O.batch_grad(p, O.u8_to_f32(d["train_u8"][base:base + cnt]), d["train_labels"][base:base + cnt])
        else:
            g, es = np.zeros(O.NPARAM), 0.0
        packed = torch.from_numpy(np.concatenate([g, [es]]))
        dist.all_reduce(packed)                      # the single exchange of the step
        lr = np.float32(0.1) / np.float32(S.effective_global_batch(cursor, B, world, n))
        p = O.apply_update(p, packed.numpy()[:O.NPARAM].astype(np.float32), lr)
        cursor = S.next_cursor(cursor, B, world, n)
    q.put((rank, p))
    dist.destroy_process_group()


def test_data_parallel_two_ranks_equal_single_process_gloo():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, q)) for r in range(2)]
    for pr in procs:
        pr.start()
    res = dict(q.get(timeout=120) for _ in range(2))
    for pr in procs:
        pr.join(timeout=60)
        assert pr.exitcode == 0
    # replicas identical
    assert np.array_equal(res[0].view(np.uint32), res[1].view(np.uint32))
    # and equal to one process doing the global batches
    d = np.load(os.path.join(O.GOLDEN, "mnist_subset.npz"))
    p = O.init_params()
    for lo in (0, 32, 64):
        hi = min(80, lo + 32)
        g, _ = O.batch_grad(p, O.u8_to_f32(d["train_u8"][lo:hi]), d["train_labels"][lo:hi])
        p = O.apply_update(p, g.astype(np.float32), np.float32(0.1) / np.float32(hi - lo))
    np.testing.assert_allclose(res[0], p, rtol=1e-6, atol=1e-7)


def test_conv_backward_tile_planning_is_host_logic(pkg):
    """pcnn_conv_bwd_plan_info needs no GPU: the tile shapes DESIGN.md 3.7 quotes for BASELINE config 5, and the shapes that must
    are refused (the FMA-pipe reference kernels run only after pcnn_conv_bwd_select)."""
    import ctypes as C

    def info(*shape):
        out = (C.c_int * 9)()
        assert pkg.lib().pcnn_conv_bwd_plan_info(*shape, out) == 0
        return list(out)

    cfg5 = info(128, 224, 224, 3, 64, 3, 3)
    assert cfg5[:4] == [1, 3, 112, 3]            # weight gradient: 3 dy rows x 112 pixels per tile (222 = 74 x 3, 2 x 112 >= 222), 3 stages
    assert cfg5[4:8] == [1, 2, 28, 3]            # input gradient: 2 strips of 112 columns, 28 outputs per lane quarter, 3 partial rows
    assert cfg5[8] >= 8
    k128 = info(4, 64, 64, 3, 128, 3, 3)
    assert k128[0] == 1 and k128[1] <= 2 and k128[4] == 1          # N = RB * 128 <= 256
    lenet = info(4, 28, 28, 1, 6, 5, 5)          # LeNet c1: 6 filters are zero-padded to 64 and run on the tensor-core kernels
    assert lenet[0] == 1 and lenet[4] == 1        # (given a row pitch that is a multiple of 8 elements)
    assert info(1, 32, 32, 3, 320, 3, 3)[0] == 0 and info(1, 32, 32, 3, 320, 3, 3)[4] == 0   # more than 256 filters: refused
    assert info(1, 32, 32, 3, 64, 5, 5)[0] == 0 and info(1, 32, 32, 3, 64, 5, 5)[4] == 1    # 5x5x3: 75 Hankel rows > 64


def test_bench_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` (the driver's reference arm) runs on host cores only and prints ONE JSON line with the keys the
    contract names; under torchrun only rank 0 prints."""
    import json
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, RANK="0", WORLD_SIZE="1")
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0", "--gpus", "1"],
                       capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "MNIST training images/sec" and d["unit"] == "images/s"
    assert d["higher_is_better"] is True and d["value"] > 100.0 and d["gpu_launches"] == 0
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"] == {"value": d["value"], "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    r1 = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0", "--gpus", "2"],
                        capture_output=True, text=True, timeout=120, env=dict(os.environ, RANK="1", WORLD_SIZE="2"))
    assert r1.returncode == 0 and r1.stdout.strip() == ""


def test_forward_conv_plan_query_is_host_logic(pkg):
    """pcnn_conv_tc_plan_info needs no GPU and no context: the tiling pcnn_conv_tc_plan_create_strided uses, and the same refusals."""
    cfg5 = pkg.conv_tc_plan_info(128, 224, 224, 3, 64, 3, 3)
    assert cfg5 == dict(Qt=4, V=2, stages=4, n_mtiles=224, n_qtiles=56, tiles=12544)     # 128 * 224 rows / 128; 222 = 55 x 4 + 2
    lenet = pkg.conv_tc_plan_info(8192, 28, 28, 1, 6, 5, 5, row_pitch=32, image_rows=32)
    assert (lenet["Qt"], lenet["V"], lenet["n_mtiles"], lenet["n_qtiles"]) == (24, 1, 2048, 1)
    s2 = pkg.conv_tc_plan_info(64, 224, 224, 3, 64, 3, 3, stride=2)
    assert s2["n_mtiles"] == 64 * 112 // 128 and s2["n_qtiles"] == -(-111 // s2["Qt"])
    for bad in [dict(C=64), dict(row_pitch=28, C=1), dict(stride=5), dict(image_rows=27, C=1)]:
        a = dict(N=1, H=28, W=28, C=3, K=64, R=3, S=3, stride=1, row_pitch=None, image_rows=0)
        a.update(bad)
        with pytest.raises(pkg.PcnnError):
            pkg.conv_tc_plan_info(**a)


@pytest.mark.parametrize("sm_count", [114, 132])
def test_multi_tile_conv_cases_reach_their_regime(pkg, sm_count):
    """The multi-tile cases of test_conv_tc_gpu.py on an H100 PCIe (114 SMs) and SXM (132 SMs), from the host-side plan queries:
    forward / weight gradient run more than 2 x stages tiles on every CTA (the stage ring wraps at least twice); the input
    gradient has more rows per share than stages and shares that cross an image boundary; the padding cases of the weight
    gradient walk a CTA through several pixel chunks with a ragged last row block."""
    import conv_ref as CR
    for N, H, W, C, K, R, S, stride, pitch, rows, _ in CR.FWD_MULTI:
        g = CR.fwd_regime(pkg, N, H, W, C, K, R, S, sm_count, stride, pitch, rows)
        assert g["min_tiles_per_cta"] > 2 * g["stages"], g
    seen = dict(ragged=0, chunks=0, dgrad_only=0)
    for N, H, W, C, K, R, S, _, _ in CR.BWD_MULTI + CR.WGRAD_PAD:
        w, d = CR.wgrad_regime(pkg, N, H, W, C, K, R, S, sm_count), CR.dgrad_regime(pkg, N, H, W, C, K, R, S, sm_count)
        assert d["max_rows_per_share"] > d["stages"] and d["shares_crossing_images"] > 0, d
        if w is None:
            seen["dgrad_only"] += 1
            continue
        assert w["min_tiles_per_cta"] > 2 * w["stages"], w
        seen["ragged"] += w["ragged"]
        seen["chunks"] += w["n_ch"] >= 2
    assert seen["ragged"] >= 3 and seen["chunks"] >= 2 and seen["dgrad_only"] == 2, seen
    w = CR.wgrad_regime(pkg, *CR.WGRAD_PAD[0][:7], sm_count)
    assert w["ragged"] and math.gcd(w["n_ch"], w["grid"]) == 1     # consecutive tiles of a CTA (grid apart) change chunk
