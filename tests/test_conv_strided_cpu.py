"""Host-side checks of the strided backward passes (no GPU): the float64 references against a direct-loop oracle, the plan
query at stride 1 against the stride-1 query, the regime every BWD_STRIDED_MULTI case reaches, and the stride refusals."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import conv_ref as CR
import conv_ref_strided as CS
import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def strided_oracle(tmp_path_factory):
    """tests/strided_bwd_oracle.c built with the oracle's parity flags (oracle/Makefile) into a temporary directory"""
    cc = os.environ.get("CC") or shutil.which("gcc") or shutil.which("cc")
    assert cc, "a C compiler is needed to build the strided backward oracle"
    so = str(tmp_path_factory.mktemp("oracle") / "libstrided_bwd_oracle.so")
    subprocess.run([cc, "-O2", "-ffp-contract=off", "-fPIC", "-std=c99", "-Wall", "-shared", "-o", so,
                    os.path.join(HERE, "strided_bwd_oracle.c")], check=True)
    L = C.CDLL(so)
    f = C.POINTER(C.c_float)
    L.orc_conv_wgrad_nhwc_strided.argtypes = [f, f, f] + [C.c_int] * 8
    L.orc_conv_dgrad_nhwc_strided.argtypes = [f, f, f] + [C.c_int] * 8
    return L


STRIDED_REF_SHAPES = [  # N, H, W, C, K, R, S, stride
    (2, 9, 11, 1, 6, 3, 3, 1), (2, 12, 10, 2, 16, 5, 5, 2), (1, 13, 14, 3, 64, 7, 7, 3), (2, 8, 9, 4, 96, 3, 3, 2),
    (1, 10, 12, 8, 64, 5, 5, 2), (3, 7, 8, 8, 64, 3, 3, 3), (2, 15, 13, 1, 96, 3, 3, 4), (2, 11, 14, 3, 32, 3, 3, 4),
]


def _within_one_ulp(ref64, got32):
    r = ref64.astype(np.float32)
    return np.all(np.abs(r - got32) <= np.spacing(np.maximum(np.abs(r), np.abs(got32))))


@pytest.mark.parametrize("shape", STRIDED_REF_SHAPES, ids=["x".join(map(str, s)) for s in STRIDED_REF_SHAPES])
def test_strided_float64_backward_references_match_the_c_oracle(strided_oracle, shape):
    """conv_wgrad_f64 / conv_dgrad_f64 with a stride against the direct loops of strided_bwd_oracle.c: the same sums in float64
    in another order, so they agree within 1 fp32 ulp.  At stride 1 they also equal conv_ref's stride-1 references."""
    N, H, W, C_, K, R, S, st = shape
    rng = np.random.default_rng(sum(shape))
    P, Q = CS.out_size(H, W, R, S, st)
    x = rng.uniform(0, 1, (N, H, W, C_)).astype(np.float32)
    f = rng.uniform(-0.5, 0.5, (K, R, S, C_)).astype(np.float32)
    dy = rng.uniform(-1, 1, (N, P, Q, K)).astype(np.float32)
    dw = np.empty((K, R, S, C_), np.float32)
    dx = np.full((N, H, W, C_), np.nan, np.float32)
    strided_oracle.orc_conv_wgrad_nhwc_strided(O.fp(x.reshape(-1)), O.fp(dy.reshape(-1)), O.fp(dw.reshape(-1)), N, H, W, C_, K, R, S, st)
    strided_oracle.orc_conv_dgrad_nhwc_strided(O.fp(dy.reshape(-1)), O.fp(f.reshape(-1)), O.fp(dx.reshape(-1)), N, H, W, C_, K, R, S, st)
    assert _within_one_ulp(CS.conv_wgrad_f64(x, dy, R, S, st), dw)
    assert _within_one_ulp(CS.conv_dgrad_f64(dy, f, H, W, st), dx)
    if st == 1:
        assert np.array_equal(CS.conv_wgrad_f64(x, dy, R, S), CR.conv_wgrad_f64(x, dy, R, S))
        assert np.array_equal(CS.conv_dgrad_f64(dy, f, H, W), CR.conv_dgrad_f64(dy, f))


def test_strided_dgrad_reference_zeroes_uncovered_rows_and_columns():
    """stride 4 > R = 3 and (H-R) % 4 != 0: rows and columns no window covers are exactly 0"""
    N, H, W, C_, K, R, S, st = 1, 12, 13, 1, 8, 3, 3, 4
    P, Q = CS.out_size(H, W, R, S, st)
    rng = np.random.default_rng(5)
    dx = CS.conv_dgrad_f64(rng.uniform(-1, 1, (N, P, Q, K)), rng.uniform(0.5, 1, (K, R, S, C_)), H, W, st)
    covered_h = np.zeros(H, bool)
    covered_w = np.zeros(W, bool)
    for p in range(P):
        covered_h[p * st:p * st + R] = True
    for q in range(Q):
        covered_w[q * st:q * st + S] = True
    assert not covered_h.all() and not covered_w.all()
    assert np.all(dx[:, ~covered_h] == 0) and np.all(dx[:, :, ~covered_w] == 0)


def test_bwd_plan_info_strided_at_stride_1_equals_the_stride_1_query(pkg):
    """pcnn_conv_bwd_plan_info_strided(..., 1, out) is pcnn_conv_bwd_plan_info for every multi-tile and tensor-core shape"""
    import test_conv_tc_gpu as G
    shapes = [c[:7] for c in CR.BWD_MULTI] + [tuple(s[:7]) for s in G.BWD_TC_SHAPES]
    L = pkg.lib()
    for shape in shapes:
        a, b = (C.c_int * 9)(), (C.c_int * 9)()
        assert L.pcnn_conv_bwd_plan_info(*shape, a) == 0
        assert L.pcnn_conv_bwd_plan_info_strided(*shape, 1, b) == 0
        assert list(a) == list(b), shape


@pytest.mark.parametrize("sm_count", CR.SM_COUNTS)
def test_strided_multi_tile_cases_reach_their_regime(pkg, sm_count):
    """Every BWD_STRIDED_MULTI case drives the kernels through their stage rings on 114- and 132-SM parts: more than 2 x stages
    tiles on every weight-gradient CTA, and input-gradient shares longer than the stage ring that cross images."""
    ragged = 0
    for N, H, W, C_, K, R, S, st, pitch, rows in CS.BWD_STRIDED_MULTI:
        w = CS.wgrad_regime(pkg, N, H, W, C_, K, R, S, sm_count, st)
        d = CS.dgrad_regime(pkg, N, H, W, C_, K, R, S, sm_count, st)
        if w is not None:
            assert w["min_tiles_per_cta"] > 2 * w["stages"], (st, w)
            ragged += w["ragged"]
        assert d is not None, "every case has a tensor-core input gradient"
        assert d["max_units_per_share"] > d["stages"] and d["shares_crossing_images"] > 0, (st, d)
        assert d["ring"] == st * ((R - 1) // st + 1)
    assert ragged >= 2
    assert sum(CS.wgrad_regime(pkg, *c[:7], sm_count, c[7]) is None for c in CS.BWD_STRIDED_MULTI) >= 1


def test_strided_backward_refuses_strides_outside_1_to_4(pkg):
    """stride 0 and 5 are PCNN_ERR_ARG, from the plan query as from the entry points (checked before any device work)"""
    for st in (0, 5):
        with pytest.raises(pkg.PcnnError, match="stride"):
            pkg.conv_bwd_plan_info(8, 28, 28, 1, 64, 3, 3, st)
        L = pkg.lib()
        for fn in (L.pcnn_conv_wgrad_strided, L.pcnn_conv_dgrad_strided):
            assert fn(None, None, None, None, 8, 28, 28, 1, 64, 3, 3, st, 0, 0) != 0     # NULL context: refused, nothing runs
    b = pkg.conv_bwd_plan_info(128, 224, 224, 3, 64, 3, 3, 2)
    assert b["wgrad_tc"] and b["dgrad_tc"] and b["dgrad_ring"] == 4
