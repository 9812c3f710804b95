"""GPU tests of the LeNet kernels whose grid is capped, at batch sizes where their loop over images or elements runs a second
time: the evaluation pass (pcnn_forward_batch, pcnn_test), the LeNet-5 variant (pcnn_l5_*), the batched operator tier and the
planar extension ops (max pool, softmax cross-entropy).  The grid rules and batch sizes are in tests/laps_ref.py; every test
first asserts the regime it claims for the running device and prints grid, laps and the worst ratio to each bound.

Batches larger than the 1024 golden digits tile them, so image (row, sample) i and i mod 1024 must give bit-identical results,
whichever CTA, thread and lap ran them.  Bounds are those of the first-lap tests (test_fused_gpu.py, test_lenet5_gpu.py,
test_ops_gpu.py, test_ext_gpu.py):
  evaluation     f_out |d| <= 1e-6 + 1e-5 |ref|; bit-identical to one image per CTA, u8 == f32; pred = first argmax of f_out
  LeNet-5        gradient rel-L2 <= 1e-5 (each block <= 2e-5), error sum within 1e-5 relative; forward as the evaluation pass
  operators      element-wise ops bit-identical to the oracle records, except that the sigmoid may differ by SIG_ULPS ulp
                 (the ops that apply it to a gradient must equal the float32 replay on such a sigmoid); batch sums
                 bit-identical to float32 of the sequential float64 sum of the per-sample float32 values
  extension      max pool bit-exact; softmax-CE within 1e-6 of the oracle
"""
import numpy as np
import pytest

import laps_ref as LR
import oracle_lib as O

pytestmark = pytest.mark.gpu
NB = LR.NB
SIG_ULPS = 1
NOUT = 7354                      # f.output inside the oracle's activation record


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def tile(a, B):
    """rows i mod len(a) for i < B"""
    return np.ascontiguousarray(a[np.arange(B) % len(a)])


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def out_ratio(got, ref):
    """worst |got - ref| / (1e-6 + 1e-5 |ref|)"""
    ref = np.asarray(ref, np.float64)
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / (1e-6 + 1e-5 * np.abs(ref))))


def at(d, i):
    """device address of row i of the DeviceArray d"""
    return d.ptr + i * (d.nbytes // d.shape[0])


@pytest.fixture(scope="module")
def sm(eng):
    return eng.device_info()["sm_count"]


@pytest.fixture(scope="module")
def digits(golden):
    u8 = golden["train_u8"][:NB]
    assert u8.shape == (NB, 784)
    return dict(u8=u8, f32=O.u8_to_f32(u8), labels=golden["train_labels"][:NB])


# ==================================================================================== 1. evaluation pass
@pytest.fixture(scope="module")
def eval_ref(golden, digits):
    p = golden["params_after1000"]
    return p, np.stack([O.forward(p, digits["f32"][i])[NOUT:] for i in range(NB)])


@pytest.mark.parametrize("case", range(4), ids=["cap+1", "2cap+7", "1024", "8192tiled"])
def test_forward_batch_past_the_first_lap(eng, pkg, sm, digits, eval_ref, case):
    p, ref = eval_ref
    B, need = LR.eval_batches(sm)[case]
    grid = LR.fused_grid(sm, B)
    fewest, most = LR.images_per_cta(B, grid)
    assert most >= need, (B, grid, most)
    eng.set_params(p)
    d8, d32 = eng.to_device(tile(digits["u8"], B)), eng.to_device(tile(digits["f32"], B))
    res = {}
    for name, d, pt in (("u8", d8, pkg.U8), ("f32", d32, pkg.F32)):
        f, pr = eng.array((B, 10)), eng.array(B, np.uint8)
        eng.forward_batch(d, pt, B, f, pr)
        res[name] = f.to_host(), pr.to_host()
    f, pred = res["u8"]
    assert np.array_equal(bits(res["f32"][0]), bits(f)) and np.array_equal(res["f32"][1], pred)
    # the same images in chunks of at most one image per CTA
    cap = LR.fused_grid(sm, 1 << 30)
    fc, pc = eng.array((B, 10)), eng.array(B, np.uint8)
    for lo in range(0, B, cap):
        eng.forward_batch(at(d8, lo), pkg.U8, min(cap, B - lo), at(fc, lo), at(pc, lo))
    assert np.array_equal(bits(fc.to_host()), bits(f)) and np.array_equal(pc.to_host(), pred)
    base = np.arange(B) % NB
    assert np.array_equal(bits(f), bits(f[base]))                 # tiled images: the same bits as their base image
    r = ref[base]
    ratio = out_ratio(f, r)
    assert ratio <= 1.0
    assert np.array_equal(pred, np.argmax(f, axis=1))             # first maximum of the device's own outputs
    top = np.sort(r, axis=1)
    wide = top[:, -1] - top[:, -2] > (2e-6 + 1e-5 * (np.abs(top[:, -1]) + np.abs(top[:, -2])))
    assert np.array_equal(pred[wide], np.argmax(r, axis=1)[wide])
    close = int(np.count_nonzero(~wide))
    assert close * 100 <= B, close
    print(f"\nforward_batch B={B} grid={grid} images per CTA {fewest}..{most}: worst |d|/bound {ratio:.3g}, "
          f"{close} images with the oracle's top two closer than their bounds")
    for a in (d8, d32, fc, pc):
        a.free()


@pytest.mark.parametrize("B", [NB, 8 * NB])
def test_test_counts_what_forward_batch_misclassifies(eng, pkg, sm, golden, digits, B):
    grid = LR.fused_grid(sm, B)
    fewest, most = LR.images_per_cta(B, grid)
    assert most >= 3, (B, grid)
    eng.set_params(golden["params_after1000"])
    imgs, labs = tile(digits["u8"], B), tile(digits["labels"], B)
    d, pr = eng.to_device(imgs), eng.array(B, np.uint8)
    eng.forward_batch(d, pkg.U8, B, None, pr)
    wrong = int(np.count_nonzero(pr.to_host() != labs))
    for pixels in (imgs, tile(digits["f32"], B)):
        eng.dataset_upload(pkg.TEST_SET, pixels, labs)
        assert eng.test() == wrong
        assert eng.test() == wrong                                # the counter is reset for every call
    print(f"\ntest() B={B} grid={grid} images per CTA {fewest}..{most}: {wrong} wrong")
    d.free(); pr.free()


# ==================================================================================== 2. LeNet-5 variant
def l5_grads(eng, pkg, p_dev, imgs, pixel_type, labs_dev, B):
    dg = eng.array((O.L5_NPARAM + 1,))
    eng.l5_compute_grads(p_dev, imgs, pixel_type, labs_dev, B, dg)
    g = dg.to_host()
    dg.free()
    return g


@pytest.mark.parametrize("case", range(3), ids=["cap+1", "2cap-1", "1024"])
def test_lenet5_gradient_past_the_first_lap(eng, pkg, sm, digits, case):
    B, need = LR.l5_batches(sm)[case]
    grid = LR.l5_grid(sm, B)
    fewest, most = LR.images_per_cta(B, grid)
    assert most >= need and B <= NB, (B, grid, most)
    p = O.l5_init_params(11)
    g_ref, err_ref = O.l5_batch_grad(p, digits["f32"][:B], digits["labels"][:B])
    dp_, dl = eng.to_device(p), eng.to_device(digits["labels"][:B])
    d8, d32 = eng.to_device(digits["u8"][:B]), eng.to_device(digits["f32"][:B])
    got = l5_grads(eng, pkg, dp_, d8, pkg.U8, dl, B)
    r = rel_l2(got[:O.L5_NPARAM], g_ref)
    assert r <= 1e-5
    blocks = {name: rel_l2(got[lo:hi], g_ref[lo:hi]) / 2e-5 for name, (lo, hi) in O.L5_OFF.items()}
    assert max(blocks.values()) <= 1.0, blocks
    e = abs(got[O.L5_NPARAM] - err_ref) / (1e-5 * err_ref)
    assert e <= 1.0
    assert np.array_equal(bits(l5_grads(eng, pkg, dp_, d8, pkg.U8, dl, B)), bits(got))      # rerun
    assert np.array_equal(bits(l5_grads(eng, pkg, dp_, d32, pkg.F32, dl, B)), bits(got))    # fp32 pixels
    worst = max(blocks, key=blocks.get)
    print(f"\nl5 gradient B={B} grid={grid} images per CTA {fewest}..{most}: rel-L2/1e-5 {r / 1e-5:.3g}, "
          f"worst block {worst} {blocks[worst]:.3g}, error sum {e:.3g}")


def test_lenet5_gradient_at_8192_tiled_is_eight_times_1024(eng, pkg, sm, digits):
    B = 8 * NB
    grid = LR.l5_grid(sm, B)
    fewest, most = LR.images_per_cta(B, grid)
    assert most >= 3, (B, grid)
    p = O.l5_init_params(11)
    dp_ = eng.to_device(p)
    d, dl = eng.to_device(tile(digits["u8"], B)), eng.to_device(tile(digits["labels"], B))
    g = l5_grads(eng, pkg, dp_, d, pkg.U8, dl, B)
    assert np.array_equal(bits(l5_grads(eng, pkg, dp_, d, pkg.U8, dl, B)), bits(g))
    g1 = l5_grads(eng, pkg, dp_, d, pkg.U8, dl, NB)                # the first NB images are the fixture
    r = rel_l2(g[:O.L5_NPARAM], 8.0 * g1[:O.L5_NPARAM].astype(np.float64))
    e = abs(float(g[O.L5_NPARAM]) - 8.0 * float(g1[O.L5_NPARAM])) / (1e-5 * 8.0 * float(g1[O.L5_NPARAM]))
    assert r <= 1e-5 and e <= 1.0
    print(f"\nl5 gradient B={B} grid={grid} images per CTA {fewest}..{most}: rel-L2 to 8 x B={NB} / 1e-5 {r / 1e-5:.3g}, "
          f"error sum {e:.3g}")


def test_lenet5_train_steps_past_the_first_lap(eng, pkg, sm, digits):
    B = LR.l5_batches(sm)[0][0]
    grid = LR.l5_grid(sm, B)
    fewest, most = LR.images_per_cta(B, grid)
    assert most >= 2, (B, grid)
    imgs, labs = tile(digits["u8"], 2 * NB), tile(digits["labels"], 2 * NB)
    f32 = tile(digits["f32"], 2 * NB)
    p = O.l5_init_params(5)
    dp_, q = eng.to_device(p), p
    for lo in range(0, 4 * B, B):
        eng.l5_train_step(dp_, eng.to_device(imgs[lo:lo + B]), pkg.U8, eng.to_device(labs[lo:lo + B]), B)
        g, _ = O.l5_batch_grad(q, f32[lo:lo + B], labs[lo:lo + B])
        q = O.l5_apply_update(q, g.astype(np.float32), np.float32(0.1) / np.float32(B))
    r = rel_l2(dp_.to_host(), q)
    assert r <= 1e-5
    print(f"\nl5 train 4 steps B={B} grid={grid} images per CTA {fewest}..{most}: parameter rel-L2/1e-5 {r / 1e-5:.3g}")


@pytest.fixture(scope="module")
def l5_out_ref(digits):
    p = O.l5_init_params(5)
    return p, np.stack([O.l5_forward_out(p, digits["f32"][i]) for i in range(NB)])


@pytest.mark.parametrize("B", [NB, 8 * NB])
def test_lenet5_forward_past_the_first_lap(eng, pkg, sm, digits, l5_out_ref, B):
    p, ref = l5_out_ref
    grid = LR.l5_grid(sm, B)
    fewest, most = LR.images_per_cta(B, grid)
    assert most >= 3, (B, grid)
    dp_ = eng.to_device(p)
    d8, d32 = eng.to_device(tile(digits["u8"], B)), eng.to_device(tile(digits["f32"], B))
    out, o32, oc = eng.array((B, 10)), eng.array((B, 10)), eng.array((B, 10))
    eng.l5_forward(dp_, d8, pkg.U8, B, out)
    eng.l5_forward(dp_, d32, pkg.F32, B, o32)
    cap = LR.l5_grid(sm, 1 << 30)
    for lo in range(0, B, cap):                                    # one image per CTA
        eng.l5_forward(dp_, at(d8, lo), pkg.U8, min(cap, B - lo), at(oc, lo))
    got = out.to_host()
    assert np.array_equal(bits(oc.to_host()), bits(got)) and np.array_equal(bits(o32.to_host()), bits(got))
    base = np.arange(B) % NB
    assert np.array_equal(bits(got), bits(got[base]))
    ratio = out_ratio(got, ref[base])
    assert ratio <= 1.0
    print(f"\nl5 forward B={B} grid={grid} images per CTA {fewest}..{most}: worst |d|/bound {ratio:.3g}")
    for a in (d8, d32, out, o32, oc):
        a.free()


# ==================================================================================== 3. batched operator tier
@pytest.fixture(scope="module")
def records(golden, digits):
    """The oracle's forward / backward record of every fixture digit with the seed-1 parameters, by field name."""
    p = golden["params_init"]
    acts = np.stack([O.forward(p, digits["f32"][s]) for s in range(NB)])
    backs = np.stack([O.backward(p, digits["f32"][s], int(digits["labels"][s]), acts[s]) for s in range(NB)])
    rec = {k: np.ascontiguousarray(acts[:, lo:hi]) for k, (lo, hi) in O.ACT_OFF.items()}
    rec.update({k: np.ascontiguousarray(backs[:, lo:hi]) for k, (lo, hi) in O.BACK_OFF.items()})
    rec.update(img=digits["f32"], labels=np.ascontiguousarray(digits["labels"]), p=p)
    # fp_preact_f on its own (the record holds it with the bias added): the kernel's sequential fp32 sum, replayed
    w = p[173:2333].reshape(10, 216)
    pre = np.zeros((NB, 10), np.float32)
    for k in range(216):
        pre = pre + w[:, k][None, :] * rec["s1_out"][:, k:k + 1]
    assert np.array_equal(bits(pre + p[2333:2343]), bits(rec["f_pre"]))
    rec["f_preact"] = pre
    return rec


def ulp_step(a, k):
    """a moved by k fp32 ulps"""
    for _ in range(abs(k)):
        a = np.nextafter(a, np.float32(np.inf if k > 0 else -np.inf)).astype(np.float32)
    return a


def preact_candidates(op, rec):
    """the float32 replays of bp_preact_* on every sigmoid within SIG_ULPS of the oracle's (layer.h:260-270, 348-369)"""
    one = np.float32(1)
    if op == "bp_preact_c1":
        dout, s = rec["c1_dout"], rec["c1_out"]
        f = lambda s: dout * (s * (one - s))
    else:
        dout, s = rec["s1_dout"], rec["s1_out"]
        f = lambda s: (dout * s) * (one - s)
    cands = [f(ulp_step(s, k)) for k in range(-SIG_ULPS, SIG_ULPS + 1)]
    assert np.array_equal(bits(cands[SIG_ULPS]), bits(rec["c1_dpre" if op == "bp_preact_c1" else "s1_dpre"]))
    return cands


# op -> (record fields of the per-sample inputs, floats per sample of the output, call, record field of the output)
ELEMENTWISE = {
    "fp_c1": (["img"], 3456, lambda e, P, o, i, B: e.fp_c1(i[0], o, P["c1w"], P["c1b"], B), "c1_pre"),
    "apply_step_function": (["c1_pre"], 3456, lambda e, P, o, i, B: e.apply_step_function(i[0], o, B * 3456), "c1_out"),
    "bp_output_c1": (["s1_dpre"], 3456, lambda e, P, o, i, B: e.bp_output_c1(o, P["s1w"], i[0], B), "c1_dout"),
    "bp_preact_c1": (["c1_dout", "c1_pre"], 3456, lambda e, P, o, i, B: e.bp_preact_c1(o, i[0], i[1], B), "c1_dpre"),
    "fp_s1": (["c1_out"], 216, lambda e, P, o, i, B: e.fp_s1(i[0], o, P["s1w"], P["s1b"], B), "s1_pre"),
    "bp_output_s1": (["f_dpre"], 216, lambda e, P, o, i, B: e.bp_output_s1(o, P["fw"], i[0], B), "s1_dout"),
    "bp_preact_s1": (["s1_dout", "s1_pre"], 216, lambda e, P, o, i, B: e.bp_preact_s1(o, i[0], i[1], B), "s1_dpre"),
    "fp_preact_f": (["s1_out"], 10, lambda e, P, o, i, B: e.fp_preact_f(i[0], o, P["fw"], B), "f_preact"),
    "fp_bias_f": (["f_preact"], 10, lambda e, P, o, i, B: e.fp_bias_f(o, P["fb"], B), "f_pre"),       # in place
    "makeError_batch": (["f_out", "labels"], 10, lambda e, P, o, i, B: e.makeError_batch(o, i[0], i[1], B), "f_dpre"),
    "vectorNorm": (["f_dpre"], 1, lambda e, P, o, i, B: e.vectorNorm(i[0], 10, B, o), "err"),
}


def run_elementwise(eng, P, op, host_inputs, B, per_sample=False):
    """`op` over the B samples of host_inputs, as one call at batch B or (per_sample) as B calls at batch 1"""
    _, width, call, _ = ELEMENTWISE[op]
    ins = [eng.to_device(a) for a in host_inputs]
    out = eng.to_device(host_inputs[0]) if op == "fp_bias_f" else eng.array((B, width))
    if per_sample:
        for s in range(B):
            call(eng, P, at(out, s), [at(d, s) for d in ins], 1)
    else:
        call(eng, P, out, ins, B)
    got = out.to_host().reshape(B, width)
    for d in ins + [out]:
        d.free()
    return got


@pytest.fixture(scope="module")
def op_params(eng, records):
    return {k: eng.to_device(records["p"][lo:hi]) for k, (lo, hi) in O.OFF.items()}


@pytest.mark.parametrize("op", list(ELEMENTWISE))
def test_batched_elementwise_operator_past_the_first_lap(eng, records, op_params, op):
    fields, width, _, ref_field = ELEMENTWISE[op]
    B = LR.ops_batch(op)
    blocks, threads, laps = LR.ops_laps(op, B)
    assert laps >= 2, (op, B, laps)
    base = run_elementwise(eng, op_params, op, [records[f] for f in fields], NB, per_sample=True)
    ref = records[ref_field].reshape(NB, width)
    if op == "apply_step_function":
        a, b = bits(base).astype(np.int64), bits(ref).astype(np.int64)      # both positive: ulps are bit distances
        worst = int(np.max(np.abs(a - b)))
        assert worst <= SIG_ULPS
        note = f"worst {worst} ulp of {SIG_ULPS}, {np.count_nonzero(a != b)} values differ"
    elif op in ("bp_preact_c1", "bp_preact_s1"):
        cands = preact_candidates(op, records)
        assert np.all(np.any([bits(base) == bits(c) for c in cands], axis=0))
        note = f"every value a replay on a sigmoid within {SIG_ULPS} ulp, {np.count_nonzero(bits(base) != bits(ref))} differ from the oracle"
    else:
        assert np.array_equal(bits(base), bits(ref))
        note = "bit-exact to the oracle"
    got = run_elementwise(eng, op_params, op, [tile(records[f], B) for f in fields], B)
    bad = np.flatnonzero(np.any(bits(got) != bits(base[np.arange(B) % NB]), axis=1))
    assert bad.size == 0, f"{bad.size} samples differ from their batch-1 run, first {bad[:8]}"
    print(f"\n{op} B={B} blocks={blocks}x{threads} laps={laps}: every sample bit-identical to batch 1; batch 1 {note}")


# op -> (record fields of the per-sample inputs, slice of the per-sample gradient record, call, bias field and divisor or None)
REDUCTIONS = {
    "bp_weight_c1": (["c1_dpre", "img"], slice(0, 150), lambda e, o, i, B: e.bp_weight_c1(o, i[0], i[1], B), None),
    "bp_weight_s1": (["s1_dpre", "c1_out"], slice(156, 172), lambda e, o, i, B: e.bp_weight_s1(o, i[0], i[1], B), None),
    "bp_bias_c1": (["c1_dpre"], slice(150, 156), lambda e, o, i, B: e.bp_bias_c1(o, i[0], B), ("c1b", 576)),
    "bp_bias_s1": (["s1_dpre"], slice(172, 173), lambda e, o, i, B: e.bp_bias_s1(o, i[0], B), ("s1b", 216)),
}


@pytest.mark.parametrize("op", list(REDUCTIONS))
def test_batched_reduction_operator_past_the_first_lap(eng, records, op):
    fields, gs, call, bias = REDUCTIONS[op]
    B = LR.ops_batch(op)
    blocks, threads, laps = LR.ops_laps(op, B)
    assert laps >= 2, (op, B, laps)
    part = records["g"][:, gs]                                     # the per-sample fp32 values (bit-exact at batch 1, test_ops_gpu)
    total = np.cumsum(tile(part, B).astype(np.float64), axis=0)[-1].astype(np.float32)     # sequential, in sample order
    ins = [eng.to_device(tile(records[f], B)) for f in fields]
    eng.set_learning_rate(0.1)
    if bias is None:
        out = eng.array(part.shape[1])
        exp = total
    else:
        lo, hi = O.OFF[bias[0]]
        b0 = records["p"][lo:hi]
        out = eng.to_device(b0)
        step = np.float32(0.1) / np.float32(B)
        exp = b0 + (step * total) / np.float32(bias[1])
    call(eng, out, ins, B)
    got = out.to_host()
    assert np.array_equal(bits(got), bits(exp)), (got, exp)
    for d in ins + [out]:
        d.free()
    print(f"\n{op} B={B} partial blocks={blocks}x{threads} laps={laps}: bit-identical to the float64 sum of the per-sample values")


# ==================================================================================== 4. planar extension ops
@pytest.mark.parametrize("planes,H,W,k", LR.MAXPOOL_CASES)
def test_planar_maxpool_past_the_first_lap(eng, sm, planes, H, W, k):
    (gf, lf), (gb, lb) = LR.maxpool_laps(sm, planes, H, W, k)
    assert lf >= 2 and lb >= 2, (lf, lb)
    rng = np.random.default_rng(planes + k)
    x = np.ascontiguousarray((rng.integers(0, 6, planes * H * W) / 4.0).astype(np.float32))     # quantised: many ties
    n_out = planes * (H // k) * (W // k)
    out_ref, arg_ref = np.empty(n_out, np.float32), np.empty(n_out, np.int32)
    O.oracle().orc_maxpool_fwd(O.fp(x), O.fp(out_ref), O.i32p(arg_ref), planes, H, W, k)
    dx, d_out, d_arg = eng.to_device(x), eng.array(n_out), eng.array(n_out, np.int32)
    eng.maxpool_fwd(dx, d_out, d_arg, planes, H, W, k)
    assert np.array_equal(d_arg.to_host(), arg_ref)
    assert np.array_equal(bits(d_out.to_host()), bits(out_ref))
    dout = rng.standard_normal(n_out).astype(np.float32)
    din_ref = np.empty(planes * H * W, np.float32)
    O.oracle().orc_maxpool_bwd(O.fp(dout), O.i32p(arg_ref), O.fp(din_ref), planes, H, W, k)
    d_din = eng.array(planes * H * W)
    eng.maxpool_bwd(eng.to_device(dout), d_arg, d_din, planes, H, W, k)
    assert np.array_equal(bits(d_din.to_host()), bits(din_ref))
    print(f"\nmaxpool {planes}x{H}x{W} k={k}: forward grid {gf}x256 laps {lf}, backward grid {gb}x256 laps {lb}: bit-exact")
    for a in (dx, d_out, d_arg, d_din):
        a.free()


@pytest.mark.parametrize("B,n", LR.SOFTMAX_CASES)
def test_softmax_ce_past_the_first_lap(eng, sm, B, n):
    grid, rows, laps = LR.softmax_laps(sm, B)
    assert laps >= 2, (B, rows)
    rng = np.random.default_rng(B + n)
    z = (rng.standard_normal((NB, n)) * 4).astype(np.float32)
    y = rng.integers(0, n, NB).astype(np.uint8)
    prob_ref, d_ref, loss_ref = np.empty((NB, n), np.float32), np.empty((NB, n), np.float32), np.empty(NB, np.float32)
    for b in range(NB):
        loss_ref[b] = O.oracle().orc_softmax_ce(O.fp(z[b]), int(y[b]), n, O.fp(prob_ref[b]), O.fp(d_ref[b]))
    dz, dy = eng.to_device(tile(z, B)), eng.to_device(tile(y, B))
    dp, dd, dl = eng.array((B, n)), eng.array((B, n)), eng.array(B)
    eng.softmax_ce(dz, dy, B, n, dp, dd, dl)
    base = np.arange(B) % NB
    got = dict(prob=dp.to_host(), d=dd.to_host(), loss=dl.to_host())
    ratios = {}
    for name, ref, rtol in (("prob", prob_ref, 0.0), ("d", d_ref, 0.0), ("loss", loss_ref, 1e-6)):
        g = got[name]
        assert np.array_equal(bits(g), bits(g[base])), name                 # tiled rows: the bits of their base row
        r = ref[base].astype(np.float64)
        ratios[name] = float(np.max(np.abs(g - r) / (1e-6 + rtol * np.abs(r))))
        assert ratios[name] <= 1.0, name
    print(f"\nsoftmax_ce B={B} n={n} grid={grid}x256 ({rows} rows per lap) laps={laps}: worst ratio to 1e-6 "
          + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()))
    for a in (dz, dy, dp, dd, dl):
        a.free()
