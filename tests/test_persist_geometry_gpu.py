"""The persistent training kernel (csrc/persist_kernels.cu, k_train_persist) in every geometry persist_geometry launches it in,
against the float64 oracle.

One kernel, several launch classes, chosen from the batch B and the device's co-residency caps (occupancy queries, so
nothing here assumes 132 SMs):
  A  B <= SM count: one image per CTA, clusters of 8, grid = B rounded up to 8 (image_step_single)
  B  SM count < B, ceil(B / 2) rounded up to 4 within the cap of two-image CTAs in clusters of 4 (IPC = 2)
  C  the next batches, two-image CTAs in clusters of 2
  D  above that: one image per CTA, clusters of 8, grid < B; image_steps_multi while the batch outnumbers the grid, the
     single-image body on a tail batch -- both inside one launch
  E  pcnn_persist_tune bit 0: no clusters (CS = 1), owners gather up to cta_capacity slots through the phase loop
  F  pcnn_persist_tune bit 1: the same kernels launched without the cooperative attribute
Bounds: parameters after a cursor-driven trajectory rtol 2e-5, atol 2e-6 against the oracle (as the learn tests); err_sum
within 1e-5 relative; the gradient of one step at frozen weights rel-L2 <= 1e-5 overall and <= 2e-5 per block of O.OFF
(as test_step_gradient_vs_frozen_weight_oracle).  Launch split, reruns, u8 vs fp32 pixels, the non-cooperative launch and the
host-pinned pull are bit-identical: the geometry depends only on B, so the arithmetic is the same.
"""
import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu

N_FIXTURE = 1024
DT = np.float32(0.1)


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def round_up(x, m):
    return (x + m - 1) // m * m


def walk(n, B, k, cur=0):
    """(cursor, images) of k cursor-driven steps as k_train_persist walks them: nb = min(B, n - cur), then cur += B and
    cur = 0 once cur >= n."""
    out = []
    for _ in range(k):
        out.append((cur, min(B, n - cur)))
        cur += B
        if cur >= n:
            cur = 0
    return out


def split_n(B):
    """A split B does not divide (B = 1 aside) with a tail of about B / 2, at most the fixture: three full batches and a tail
    for the batches up to 341, 1024 beyond (B = 1000: a tail of 24)."""
    return 3 * B + max(B // 2, 1) if 3 * B + max(B // 2, 1) <= N_FIXTURE else N_FIXTURE


def two_passes(n, B):
    """steps of two passes over the split and one more: the tail and the wrap-around fall inside the launch"""
    return 2 * ((n + B - 1) // B) + 1


@pytest.fixture(scope="module")
def data(eng, pkg, golden):
    eng.set_learning_rate(float(DT))
    d = dict(u8=golden["train_u8"][:N_FIXTURE], labels=golden["train_labels"][:N_FIXTURE], p0=golden["params_init"])
    d["f32"] = O.u8_to_f32(d["u8"])
    d["d_f32"] = eng.to_device(d["f32"])
    d["d_labels"] = eng.to_device(d["labels"])
    return d


def upload(eng, pkg, data, n):
    eng.dataset_upload(pkg.TRAIN_SET, data["u8"][:n], data["labels"][:n])


def oracle_steps(data, p, steps):
    """float64 oracle along a cursor walk: frozen-weight batch gradient, update with dt / nb; returns (params, errors)"""
    errs = []
    for cur, nb in steps:
        g, e = O.batch_grad(p, data["f32"][cur:cur + nb], data["labels"][cur:cur + nb])
        p = O.apply_update(p, g.astype(np.float32), DT / np.float32(nb))
        errs.append(e)
    return p, errs


def run_steps(eng, data, n, B, k, split=False):
    """k persistent steps over the bound n-sample split from the initial parameters at cursor 0: one launch, or (split) k
    launches of one step each at the cursors walk() restates.  Returns (params, err_sum, gradient of the last step)."""
    eng.set_params(data["p0"])
    eng.err_sum(reset=True)
    if split:
        for cur, _ in walk(n, B, k):
            eng.train_steps(cur, B, 1)
    else:
        eng.train_steps(0, B, k)
    eng.sync()
    return eng.get_params(), eng.err_sum(), eng.get_grads()


def bind(eng, pkg, data, n, f32=False):
    """the first n samples as the training split: u8 pixels uploaded, or (f32) the fp32 device copy bound in place"""
    if f32:
        eng.dataset_bind(pkg.TRAIN_SET, data["d_f32"], pkg.F32, data["d_labels"], n)
    else:
        upload(eng, pkg, data, n)


def check_frozen_gradient(eng, data, n, B, k):
    """k - 1 steps, the parameters read back, then step k on its own: its gradient against the oracle at those parameters"""
    steps = walk(n, B, k)
    eng.set_params(data["p0"])
    if k > 1:
        eng.train_steps(0, B, k - 1)
    eng.sync()
    p = eng.get_params()
    cur, nb = steps[-1]
    eng.train_steps(cur, B, 1)
    eng.sync()
    g = eng.get_grads()
    g_ref, _ = O.batch_grad(p, data["f32"][cur:cur + nb], data["labels"][cur:cur + nb])
    assert rel_l2(g, g_ref) <= 1e-5, (B, cur, nb)
    for name, (lo, hi) in O.OFF.items():
        assert rel_l2(g[lo:hi], g_ref[lo:hi]) <= 2e-5, (B, cur, nb, name)


def last_step_k(n, B, kind):
    """smallest k >= 2 whose last step is a tail step (nb < B) or a full step"""
    for k in range(2, 4 * ((n + B - 1) // B) + 2):
        nb = walk(n, B, k)[-1][1]
        if (nb < B) == (kind == "tail"):
            return k
    raise AssertionError(f"no {kind} step for B={B}, n={n}")


# ------------------------------------------------------------------------------------------------------------ census
def classify(B, info, sm):
    if info["images_per_cta"] == 2:
        return "B" if info["cluster"] == 4 else "C"
    return "A" if B <= sm else "D"


@pytest.fixture(scope="module")
def census(eng, pkg, data):
    """One persistent step at every B from 1 to 2 x cta_capacity + 8; the geometry of each, the caps it implies, and one
    representative B per class edge."""
    upload(eng, pkg, data, N_FIXTURE)
    sm = eng.device_info()["sm_count"]
    cap = eng.persist_info()["cta_capacity"]
    eng.set_step_mode(pkg.MODE_PERSISTENT)
    geo = {}
    try:
        for B in range(1, 2 * cap + 9):
            eng.set_params(data["p0"])
            eng.train_steps(0, B, 1)
            geo[B] = eng.persist_info()
        eng.sync()
    finally:
        eng.set_step_mode(pkg.MODE_AUTO)
    capc = geo[1]["cta_capacity_clustered"]
    pair4 = max([i["grid"] for i in geo.values() if i["images_per_cta"] == 2 and i["cluster"] == 4], default=0)
    pair2 = max([i["grid"] for i in geo.values() if i["images_per_cta"] == 2 and i["cluster"] == 2], default=0)
    cls = {B: classify(B, i, sm) for B, i in geo.items()}
    by = {c: [B for B in geo if cls[B] == c] for c in "ABCD"}
    first_d = min(by["D"], default=None)
    d_grid = geo[first_d]["grid"] if first_d else None
    print(f"\npersistent geometry census: sm_count {sm}, cta_capacity {cap}, cta_capacity_clustered {capc}, "
          f"pair cap clusters of 4 {pair4} (B <= {max(by['B'], default=0)}), pair cap clusters of 2 {pair2} "
          f"(B {min(by['C'], default=0)}..{max(by['C'], default=0)}), class D from B = {first_d} at grid {d_grid}")
    edges = None
    if all(by.values()):
        last4, first2, last2 = max(by["B"]), min(by["C"]), max(by["C"])
        edges = dict(one=1, seven=7, sm=sm, pair4_first=sm + 1, pair4_first_n=sm + 2, pair4_last=last4, pair4_last_n=last4 - 1,
                     pair2_first=first2, pair2_first_n=first2 + 1, pair2_last=last2, pair2_last_n=last2 - 1, multi_first=first_d,
                     thousand=1000)
    return dict(geo=geo, sm=sm, cap=cap, capc=capc, pair=(pair4, pair2), cls=cls, by=by, edges=edges)


def test_census_invariants(census):
    geo, sm, cap, capc = census["geo"], census["sm"], census["cap"], census["capc"]
    pair4, pair2 = census["pair"]
    for c in "ABCD":      # a device that collapses a class is a finding, not a skip
        assert census["by"][c], f"class {c} never launched: {census['pair']}, sm {sm}, cap {cap}"
    assert pair4 % 4 == 0 and pair2 % 2 == 0 and pair4 <= sm and pair2 <= sm, census["pair"]
    assert capc % 8 == 0 and capc <= cap
    for B, i in geo.items():
        g, cs, ipc = i["grid"], i["cluster"], i["images_per_cta"]
        assert g % cs == 0, (B, i)
        assert i["cooperative"], (B, i)
        g4, g2 = round_up((B + 1) // 2, 4), round_up((B + 1) // 2, 2)
        pair = B > sm and (g4 <= pair4 or g2 <= pair2)
        assert (ipc == 2) == pair, (B, i)
        if ipc == 2:
            assert (g, cs) == ((g4, 4) if g4 <= pair4 else (g2, 2)), (B, i)
        if ipc == 1 and B <= capc:
            assert (g, cs) == (round_up(B, 8), 8), (B, i)
        if census["cls"][B] == "D":
            want = min(B, cap)
            gd = min(round_up(want, 8), capc)
            exp = (gd, 8) if gd >= want or gd * 8 >= want * 7 else (want, 1)
            assert (g, cs) == exp, (B, i)
        else:
            assert g * ipc >= B, (B, i)
    # the classes are contiguous ranges in the order A, B, C, D
    order = "".join(census["cls"][B] for B in sorted(geo))
    assert order == "".join(c * len(census["by"][c]) for c in "ABCD"), order
    first_d = min(census["by"]["D"])
    assert geo[first_d]["grid"] < first_d and geo[first_d]["grid"] * 2 > first_d     # most CTAs one image, a few two


EDGES = ["one", "seven", "sm", "pair4_first", "pair4_first_n", "pair4_last", "pair4_last_n", "pair2_first", "pair2_first_n",
         "pair2_last", "pair2_last_n", "multi_first", "thousand"]
EDGE_CLASS = dict(one="A", seven="A", sm="A", pair4_first="B", pair4_first_n="B", pair4_last="B", pair4_last_n="B", pair2_first="C",
                  pair2_first_n="C", pair2_last="C", pair2_last_n="C", multi_first="D", thousand="D")


def edge_b(census, edge):
    assert census["edges"] is not None, "the census did not find every class"
    B = census["edges"][edge]
    if B <= 2 * census["cap"] + 8:
        assert census["cls"][B] == EDGE_CLASS[edge], (edge, B, census["cls"][B])
    return B


# ------------------------------------------------------------------------------------------------- oracle trajectories
@pytest.mark.parametrize("edge", EDGES)
def test_trajectory_matches_oracle(eng, pkg, data, census, edge):
    """train_steps over two passes and a step in one launch: tails and wrap-around inside the launch"""
    B = edge_b(census, edge)
    n = split_n(B)
    k = two_passes(n, B)
    bind(eng, pkg, data, n)
    eng.set_step_mode(pkg.MODE_PERSISTENT)
    try:
        p, err, _ = run_steps(eng, data, n, B, k)
        info = eng.persist_info()
    finally:
        eng.set_step_mode(pkg.MODE_AUTO)
    assert classify(B, info, census["sm"]) == EDGE_CLASS[edge], info
    steps = walk(n, B, k)
    if EDGE_CLASS[edge] == "D":      # both bodies in one launch: full batches above the grid, a tail within it
        assert any(nb > info["grid"] for _, nb in steps) and any(nb <= info["grid"] for _, nb in steps), (steps, info)
    p_ref, errs = oracle_steps(data, data["p0"], steps)
    np.testing.assert_allclose(p, p_ref, rtol=2e-5, atol=2e-6)
    assert abs(err - sum(errs)) <= 1e-5 * sum(errs)


@pytest.mark.parametrize("edge,kind", [(e, k) for e in EDGES for k in ("tail", "full") if (e, k) != ("one", "tail")])   # B = 1: no tail
def test_frozen_weight_gradient_of_last_step(eng, pkg, data, census, edge, kind):
    B = edge_b(census, edge)
    n = split_n(B)
    bind(eng, pkg, data, n)
    eng.set_step_mode(pkg.MODE_PERSISTENT)
    try:
        check_frozen_gradient(eng, data, n, B, last_step_k(n, B, kind))
    finally:
        eng.set_step_mode(pkg.MODE_AUTO)


# -------------------------------------------------------------------------------------------------- bit-exact invariants
@pytest.mark.parametrize("edge", EDGES)
def test_launch_split_reruns_and_f32_pixels_are_bit_identical(eng, pkg, data, census, edge):
    """The same k steps as one launch, again as one launch, as k one-step launches, and on fp32 device pixels"""
    B = edge_b(census, edge)
    n = split_n(B)
    k = two_passes(n, B)
    eng.set_step_mode(pkg.MODE_PERSISTENT)
    try:
        bind(eng, pkg, data, n)
        one = run_steps(eng, data, n, B, k)
        again = run_steps(eng, data, n, B, k)
        split = run_steps(eng, data, n, B, k, split=True)
        bind(eng, pkg, data, n, f32=True)
        f32 = run_steps(eng, data, n, B, k)
    finally:
        eng.set_step_mode(pkg.MODE_AUTO)
        upload(eng, pkg, data, n)
    for name, other in (("rerun", again), ("launch split", split), ("fp32 pixels", f32)):
        assert bits_equal(one[0], other[0]), name
        assert bits_equal(one[2], other[2]), name
        assert one[1] == other[1], name


# ------------------------------------------------------------------------------------------------------- tune variants
def restore_defaults(eng, pkg):
    eng.persist_tune(0)
    eng.set_step_mode(pkg.MODE_AUTO)


def assert_defaults_back(eng):
    """persist_tune(0) is the whole state: cooperative launches again after a bit-1 run"""
    assert eng.persist_info()["cooperative"], eng.persist_info()


def class_e_bs(census):
    return [1, 64, census["cap"], census["cap"] + 1, 1000]


@pytest.mark.parametrize("pick", range(5))
def test_class_e_without_clusters_matches_oracle(eng, pkg, data, census, pick):
    B = class_e_bs(census)[pick]
    n = split_n(B)
    k = two_passes(n, B)
    bind(eng, pkg, data, n)
    eng.set_step_mode(pkg.MODE_PERSISTENT)
    eng.persist_tune(1)
    try:
        p, err, g = run_steps(eng, data, n, B, k)
        info = eng.persist_info()
        p2, err2, g2 = run_steps(eng, data, n, B, k)
        check_frozen_gradient(eng, data, n, B, last_step_k(n, B, "tail" if n % B else "full"))
        if n % B:
            check_frozen_gradient(eng, data, n, B, last_step_k(n, B, "full"))
    finally:
        restore_defaults(eng, pkg)
    assert_defaults_back(eng)
    assert info["cluster"] == 1 and info["images_per_cta"] == 1 and info["grid"] == min(B, census["cap"]), info
    assert bits_equal(p, p2) and bits_equal(g, g2) and err == err2
    p_ref, errs = oracle_steps(data, data["p0"], walk(n, B, k))
    np.testing.assert_allclose(p, p_ref, rtol=2e-5, atol=2e-6)
    assert abs(err - sum(errs)) <= 1e-5 * sum(errs)


@pytest.mark.parametrize("edge", ["seven", "pair4_first", "multi_first"])
def test_class_f_non_cooperative_is_bit_identical(eng, pkg, data, census, edge):
    B = edge_b(census, edge)
    n = split_n(B)
    k = two_passes(n, B)
    bind(eng, pkg, data, n)
    eng.set_step_mode(pkg.MODE_PERSISTENT)
    try:
        ref = run_steps(eng, data, n, B, k)
        ref_info = eng.persist_info()
        eng.persist_tune(2)
        got = run_steps(eng, data, n, B, k)
        info = eng.persist_info()
    finally:
        restore_defaults(eng, pkg)
    assert_defaults_back(eng)
    assert ref_info["cooperative"] and not info["cooperative"], (ref_info, info)
    assert (info["grid"], info["cluster"], info["images_per_cta"]) == (ref_info["grid"], ref_info["cluster"], ref_info["images_per_cta"])
    assert bits_equal(ref[0], got[0]) and bits_equal(ref[2], got[2]) and ref[1] == got[1]


# ------------------------------------------------------------------------------------------- host-pinned pull at class D
@pytest.mark.parametrize("edge", ["multi_first", "thousand"])
def test_pinned_host_pull_at_class_d(eng, pkg, data, census, edge):
    """learn_host on page-locked images: the tail step (nb <= grid) requests the next step's image a step ahead, the full
    steps do not.  Bit-identical to device-resident learn and to the staged run on pageable copies; per-step errors of one
    epoch against the oracle."""
    import torch
    B = edge_b(census, edge)
    n = split_n(B)
    imgs, labs = data["u8"][:n], data["labels"][:n]
    upload(eng, pkg, data, n)
    eng.set_params(data["p0"])
    e_dev = eng.learn(B=B, epochs=2)
    p_dev = eng.get_params()
    assert classify(B, eng.persist_info(), census["sm"]) == "D"
    hi = torch.empty((n, 784), dtype=torch.uint8, pin_memory=True)
    hl = torch.empty((n,), dtype=torch.uint8, pin_memory=True)
    hi.numpy()[:] = imgs
    hl.numpy()[:] = labs
    eng.set_params(data["p0"])
    e_pull = eng.learn_host(hi.numpy(), hl.numpy(), B=B, epochs=2)
    errs_pull = eng.step_errs().copy()
    assert bits_equal(p_dev, eng.get_params())
    assert abs(e_pull - e_dev) < 1e-6
    eng.set_params(data["p0"])
    e_staged = eng.learn_host(np.array(imgs, copy=True), np.array(labs, copy=True), B=B, epochs=2)
    assert bits_equal(p_dev, eng.get_params())
    assert bits_equal(errs_pull, eng.step_errs()) and abs(e_staged - e_pull) < 1e-6
    # one epoch: every step's error sum against the oracle
    eng.set_params(data["p0"])
    eng.learn_host(hi.numpy(), hl.numpy(), B=B, epochs=1)
    errs = eng.step_errs()
    steps = walk(n, B, (n + B - 1) // B)
    _, errs_ref = oracle_steps(data, data["p0"], steps)
    assert len(errs) == len(errs_ref)
    np.testing.assert_allclose(errs, errs_ref, rtol=1e-5, atol=0)
