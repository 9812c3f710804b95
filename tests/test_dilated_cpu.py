"""Dilated convolution on the host: the references of dilated_ref.py against torch's float64 operators, the domain of the
_dilated queries (pcnn_conv_wide_plan_info_dilated, pcnn_conv_wide_bwd_info_dilated, pcnn_dwconv_info_dilated) against the rule
pcnn.h states, the _dilated queries at dilation (1, 1) against the padded and unpadded ones, conv_layer_family's routing, and the
regime of the `conv_bench.py dilated` shapes.  No GPU."""
import itertools

import numpy as np
import pytest
import torch

import dilated_ref as D

WIDE_QUERY = "pcnn_conv_wide_plan_create_dilated"
BWD_QUERY = "pcnn_conv_wide_bwd_info_dilated"
DW_QUERY = "pcnn_dwconv_info_dilated"


def _nchw(a):
    return torch.from_numpy(np.ascontiguousarray(a)).permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).numpy()


# -------------------------------------------------------------------------------------------- wide references against torch
def _ref_cases():
    """strides 1-4, dilations 1-6, every pad 0..dil (taps - 1), 1x1 .. 7x7 and 1x7 taps; the image is the window's extent plus a
    few rows so that both ragged and exact fits occur"""
    rng = np.random.default_rng(5)
    for (R, S), st, d in itertools.product([(1, 1), (2, 2), (3, 3), (5, 5), (7, 7), (1, 7)], range(1, 5), range(1, 7)):
        dh, dw = (1, d) if (R, S) == (1, 7) else (d, d)
        for ph in range(dh * (R - 1) + 1):
            pw = min(ph, dw * (S - 1)) if (R, S) != (1, 7) else int(rng.integers(0, dw * (S - 1) + 1))
            Eh, Ew = dh * (R - 1) + 1, dw * (S - 1) + 1
            H = max(1, Eh - 2 * ph) + int(rng.integers(0, st + 2))
            W = max(1, Ew - 2 * pw) + int(rng.integers(0, st + 2))
            yield (H, W, R, S, st, ph, pw, dh, dw)


REF_CASES = list(_ref_cases())


def test_wide_references_equal_torch_float64():
    """fwd_f64, wgrad_f64 and dgrad_f64 equal torch's float64 conv2d(dilation=...), conv2d_weight and conv2d_input over the
    sweep (to 1e-12 of the magnitude: both sum the same products in different orders)"""
    rng = np.random.default_rng(0)
    N, C, K = 2, 3, 2
    for H, W, R, S, st, ph, pw, dh, dw in REF_CASES:
        x = rng.standard_normal((N, H, W, C))
        f = rng.standard_normal((K, R, S, C))
        b = rng.standard_normal(K)
        P, Q = D.out_size(H, W, R, S, st, (ph, pw), (dh, dw))
        assert P >= 1 and Q >= 1
        dy = rng.standard_normal((N, P, Q, K))
        ft = _nchw(f)
        yt = torch.nn.functional.conv2d(_nchw(x), ft, torch.from_numpy(b), st, (ph, pw), (dh, dw))
        assert yt.shape[2:] == (P, Q)
        y = D.fwd_f64(x, f, b, st, (ph, pw), (dh, dw))
        np.testing.assert_allclose(y, _nhwc(yt), rtol=0, atol=1e-12 * (1 + np.abs(y).max()))
        dwt = torch.nn.grad.conv2d_weight(_nchw(x), ft.shape, _nchw(dy), st, (ph, pw), (dh, dw))
        got = D.wgrad_f64(x, dy, R, S, st, (ph, pw), (dh, dw))
        np.testing.assert_allclose(got, _nhwc(dwt), rtol=0, atol=1e-12 * (1 + np.abs(got).max()))
        dxt = torch.nn.grad.conv2d_input((N, C, H, W), ft, _nchw(dy), st, (ph, pw), (dh, dw))
        got = D.dgrad_f64(dy, f, H, W, st, (ph, pw), (dh, dw))
        np.testing.assert_allclose(got, _nhwc(dxt), rtol=0, atol=1e-12 * (1 + np.abs(got).max()))


def test_zero_inserted_filters_are_the_dilated_convolution():
    """the undilated convolution with the filters spread to E x E (zeros between the taps) is the dilated one"""
    rng = np.random.default_rng(1)
    for H, W, R, S, st, ph, pw, dh, dw in REF_CASES[::7]:
        x = rng.standard_normal((1, H, W, 2))
        f = rng.standard_normal((2, R, S, 2))
        fz = D.zero_inserted(f, (dh, dw))
        np.testing.assert_allclose(D.fwd_f64(x, fz, None, st, (ph, pw)), D.fwd_f64(x, f, None, st, (ph, pw), (dh, dw)), atol=1e-12)


def test_dgrad_phase_taps_enumerate_every_tap_once():
    """For each phase a of dx: the kernel's walk r = rho + tstep i, dy row u - dystep i + off is exactly the set of taps r with
    r dil = a + pad (mod stride), each at dy row (stride u + a + pad - r dil) / stride; at dilation 1 it is rho = (a + pad) % st,
    off = (a + pad) // st, step st, dy step 1."""
    for st, dil, R in itertools.product(range(1, 5), range(1, 9), range(1, 8)):
        for pad in range(dil * (R - 1) + 1):
            for a in range(st):
                taps, rho, off, tstep, dystep = D.dgrad_phase_taps(a, pad, dil, st, R)
                want = [r for r in range(R) if (r * dil - a - pad) % st == 0]
                walk = [rho + tstep * i for i in range(taps)]
                assert walk == want, (st, dil, R, pad, a)
                for i, r in enumerate(walk):
                    assert (st * 7 + a + pad - r * dil) // st == 7 - dystep * i + off
                    assert (st * 7 + a + pad - r * dil) % st == 0
                if dil == 1:
                    assert (tstep, dystep) == (st, 1) and (taps == 0 or (rho, off) == ((a + pad) % st, (a + pad) // st))


# ---------------------------------------------------------------------------------------- depthwise replays against torch
DW_CASES = [  # H, W, C, R, S, stride, pad, dilation
    (13, 12, 8, 3, 3, 1, (2, 2), (2, 2)),
    (14, 15, 16, 3, 3, 2, (2, 2), (2, 2)),
    (17, 16, 5, 5, 5, 1, (4, 4), (2, 2)),
    (20, 19, 8, 3, 3, 1, (6, 6), (6, 6)),
    (11, 13, 3, 3, 3, 3, (1, 3), (2, 3)),
    (9, 25, 8, 1, 7, 1, (0, 3), (1, 3)),
    (16, 16, 24, 7, 7, 4, (5, 6), (2, 2)),
    (7, 8, 8, 3, 3, 1, (0, 0), (3, 3)),
]


@pytest.mark.parametrize("case", DW_CASES, ids=[f"{c[0]}x{c[1]}x{c[2]}-{c[3]}x{c[4]}-s{c[5]}-p{c[6]}-d{c[7]}" for c in DW_CASES])
def test_depthwise_replays_agree_with_torch(case):
    """float32 replays of y and dx agree with torch's float32 CPU conv2d(groups=C, dilation=...) within float32 rounding, with NaN
    exactly where torch has NaN (Inf and NaN in x and dy); dw_wgrad_f64 equals torch's float64 weight gradient"""
    H, W, C, R, S, st, pad, dil = case
    rng = np.random.default_rng(sum(case[:6]))
    N = 2
    x = rng.standard_normal((N, H, W, C)).astype(np.float32)
    w = rng.standard_normal((C, R, S)).astype(np.float32)
    x[0, 1, 2, 0], x[1, -1, -2, -1], x[0, -2, 0, 1 % C] = np.inf, np.nan, -np.inf
    P, Q = D.out_size(H, W, R, S, st, pad, dil)
    dy = rng.standard_normal((N, P, Q, C)).astype(np.float32)
    dy[1, 0, 0, 0] = np.inf
    wt = torch.from_numpy(w).reshape(C, 1, R, S)
    yt = _nhwc(torch.nn.functional.conv2d(_nchw(x), wt, None, st, pad, dil, groups=C))
    y = D.dw_fwd(x, w, None, st, pad, dil)
    assert y.shape == yt.shape
    assert np.array_equal(np.isnan(y), np.isnan(yt))
    fin = np.isfinite(yt)
    mag = _nhwc(torch.nn.functional.conv2d(_nchw(np.abs(np.nan_to_num(x, posinf=0, neginf=0))), wt.abs(), None, st, pad, dil, groups=C))
    assert np.all(np.abs(y[fin] - yt[fin]) <= 2 * R * S * 2.0 ** -24 * mag[fin] + 1e-30)
    assert np.array_equal(y[~fin & ~np.isnan(yt)], yt[~fin & ~np.isnan(yt)])
    dxt = _nhwc(torch.nn.grad.conv2d_input((N, C, H, W), wt, _nchw(dy), st, pad, dil, groups=C))
    dx = D.dw_dgrad(dy, w, H, W, st, pad, dil)
    assert np.array_equal(np.isnan(dx), np.isnan(dxt))
    fin = np.isfinite(dxt)
    magd = _nhwc(torch.nn.grad.conv2d_input((N, C, H, W), wt.abs(), _nchw(np.abs(np.nan_to_num(dy, posinf=0))), st, pad, dil, groups=C))
    assert np.all(np.abs(dx[fin] - dxt[fin]) <= 2 * R * S * 2.0 ** -24 * magd[fin] + 1e-30)
    xd, dyd = rng.standard_normal((N, H, W, C)), rng.standard_normal((N, P, Q, C))
    dwt = torch.nn.grad.conv2d_weight(_nchw(xd), (C, 1, R, S), _nchw(dyd), st, pad, dil, groups=C).reshape(C, R, S).numpy()
    np.testing.assert_allclose(D.dw_wgrad_f64(xd, dyd, R, S, st, pad, dil), dwt, rtol=0, atol=1e-12 * (1 + np.abs(dwt).max()))


def test_depthwise_replays_at_dilation_one_are_dwconv_ref():
    import dwconv_ref as DR
    rng = np.random.default_rng(3)
    x = rng.standard_normal((2, 9, 10, 8)).astype(np.float32)
    w = rng.standard_normal((8, 3, 3)).astype(np.float32)
    for st, ph, pw in [(1, 1, 1), (2, 0, 2), (3, 2, 1)]:
        y = D.dw_fwd(x, w, None, st, (ph, pw))
        assert np.array_equal(y.view(np.uint32), DR.fwd(x, w, None, st, ph, pw).view(np.uint32))
        dy = rng.standard_normal(y.shape).astype(np.float32)
        assert np.array_equal(D.dw_dgrad(dy, w, 9, 10, st, (ph, pw)).view(np.uint32), DR.dgrad(dy, w, 9, 10, st, ph, pw)[0].view(np.uint32))


# ----------------------------------------------------------------------------------------------------- the query domains
def _wide_rule(N, H, W, C, K, R, S, st, ph, pw, dh, dw):
    """pcnn.h's domain of the _dilated wide calls, for dilations other than (1, 1) and a dense layout"""
    Eh, Ew = dh * (R - 1) + 1, dw * (S - 1) + 1
    return (1 <= st <= 4 and 1 <= R <= 7 and 1 <= S <= 7 and 1 <= dh <= 256 and 1 <= dw <= 256
            and 0 <= ph <= dh * (R - 1) and 0 <= pw <= dw * (S - 1) and N > 0 and C > 0 and K > 0
            and H + 2 * ph >= Eh and W + 2 * pw >= Ew and (ph == 0 or H >= st) and (pw == 0 or W >= st)
            and K % 8 == 0 and K <= 256 and C % 8 == 0)


def _dw_rule(N, H, W, C, R, S, st, ph, pw, dh, dw):
    Eh, Ew = dh * (R - 1) + 1, dw * (S - 1) + 1
    return (N >= 1 and H >= 1 and W >= 1 and C >= 1 and 1 <= R <= 7 and 1 <= S <= 7 and 1 <= st <= 4 and 1 <= dh <= 256
            and 1 <= dw <= 256 and 0 <= ph <= dh * (R - 1) and 0 <= pw <= dw * (S - 1) and H + 2 * ph >= Eh and W + 2 * pw >= Ew)


def _accepts(fn, *args, **kw):
    try:
        fn(*args, **kw)
        return True, ""
    except Exception as e:                                        # PcnnError
        return False, str(e)


def _sweep():
    for R, st, d in itertools.product([1, 2, 3, 5, 7, 8, 0], [1, 2, 3, 4, 5], [2, 3, 6, 256, 257, 0]):
        S = 3 if R in (0, 8) else R
        for ph in sorted({0, 1, d * (max(R, 1) - 1), d * (max(R, 1) - 1) + 1, -1}):
            for H in sorted({1, st - 1, st, d * (max(R, 1) - 1) + 1 - 2 * max(ph, 0), d * (max(R, 1) - 1) + 2 - 2 * max(ph, 0), 40}):
                if H < 1:
                    continue
                yield R, S, st, d, ph, H


def test_wide_dilated_queries_accept_exactly_the_rule(pkg):
    """Both wide _dilated queries accept exactly pcnn.h's rule over R, stride, dilation, pad and small H (W = 24, pad_w 1,
    dil_w 2, C = 64, K = 32, plus refusals of C, K); each refusal names the called function and the rule it breaks"""
    n_acc = n_ref = 0
    for R, S, st, d, ph, H in _sweep():
        for C, K in [(64, 32), (60, 32), (64, 264)]:
            args = (2, H, 24, C, K, R, S, st)
            want = _wide_rule(*args, ph, 1, d, 2)
            ok, msg = _accepts(pkg.conv_wide_plan_info, *args, padding=(ph, 1), dilation=(d, 2))
            okb, msgb = _accepts(pkg.conv_wide_bwd_info, *args, padding=(ph, 1), dilation=(d, 2))
            assert ok == want and okb == want, (args, ph, d, msg, msgb)
            if ok:
                n_acc += 1
                continue
            n_ref += 1
            assert WIDE_QUERY + ":" in msg and BWD_QUERY + ":" in msgb and msg.split(WIDE_QUERY)[-1] == msgb.split(BWD_QUERY)[-1]
            assert any(w in msg for w in ("required", "outside", "needs", "must be")), msg
    assert n_acc > 100 and n_ref > 100


def test_wide_dilated_refusals_state_their_rule(pkg):
    q = pkg.conv_wide_plan_info
    cases = [((2, 14, 14, 64, 64, 3, 3, 1), (5, 1), (2, 2), r"padding \(5, 1\) with R = 3, S = 3 taps at dilation \(2, 2\): 0 <= pad_h <= dil_h\*\(R - 1\)"),
             ((2, 4, 14, 64, 64, 3, 3, 1), (0, 1), (2, 2), r"H \+ 2\*pad_h >= dil_h\*\(R - 1\) \+ 1"),
             ((2, 3, 14, 64, 64, 3, 3, 4), (1, 1), (2, 2), r"a padded direction needs at least stride rows"),
             ((2, 14, 14, 64, 64, 3, 3, 1), (1, 1), (0, 2), r"dilation \(0, 2\): 1 <= dil_h, dil_w <= 256"),
             ((2, 14, 14, 60, 64, 3, 3, 1), (2, 2), (2, 2), r"C %? ?= ?60|C = 60 channels")]
    for args, pad, dil, pat in cases:
        with pytest.raises(pkg.PcnnError, match=WIDE_QUERY + ".*" + pat):
            q(*args, padding=pad, dilation=dil)


def test_depthwise_dilated_query_accepts_exactly_the_rule(pkg):
    for R, S, st, d, ph, H in _sweep():
        for C in (8, 5):
            args = (2, H, 17, C, R, S, st)
            want = _dw_rule(*args, ph, 2, d, 3)
            ok, msg = _accepts(pkg.dwconv_info, *args, padding=(ph, 2), dilation=(d, 3))
            assert ok == want, (args, ph, d, msg)
            if not ok:
                assert DW_QUERY + ":" in msg and "required" in msg, msg


def _strip(msg, fn):
    return msg.split(fn + ":", 1)[1]


def test_dilated_queries_at_dilation_one_are_the_padded_and_unpadded_ones(pkg):
    """At dilation (1, 1) the raw _dilated queries return the _padded queries' out8 / out10 and, for a refused shape, the same rule
    text; the _padded ones at pad 0 are the unpadded ones (a row-Toeplitz shape included).  The same for the depthwise query."""
    import ctypes
    L = pkg.lib()
    last = lambda: L.pcnn_last_error_string().decode()
    shapes = [(2, 14, 14, 64, 64, 3, 3, 1, 1, 1), (2, 13, 11, 40, 24, 5, 5, 2, 2, 2), (2, 14, 14, 64, 64, 3, 3, 1, 3, 1),
              (2, 2, 2, 64, 32, 3, 3, 4, 1, 1), (2, 8, 8, 8, 8, 3, 3, 1, 0, 0), (2, 9, 9, 64, 264, 3, 3, 1, 0, 0),
              (2, 2, 9, 64, 64, 3, 3, 1, 0, 0), (2, 20, 20, 320, 64, 7, 7, 3, 0, 0), (2, 20, 20, 64, 64, 3, 3, 5, 1, 1)]
    for N, H, W, C, K, R, S, st, ph, pw in shapes:
        base = (N, H, W, C, K, R, S, st)
        for fn_pad, fn_dil, n in [("pcnn_conv_wide_plan_info_padded", "pcnn_conv_wide_plan_info_dilated", 8),
                                  ("pcnn_conv_wide_bwd_info_padded", "pcnn_conv_wide_bwd_info_dilated", 10)]:
            a, b = (ctypes.c_int * n)(), (ctypes.c_int * n)()
            rc_p = getattr(L, fn_pad)(*base, ph, pw, W * C, 0, a)
            msg_p = last() if rc_p else ""
            rc_d = getattr(L, fn_dil)(*base, ph, pw, 1, 1, W * C, 0, b)
            msg_d = last() if rc_d else ""
            assert rc_p == rc_d, (base, fn_dil)
            if rc_p:
                name_p = "pcnn_conv_wide_plan_create_padded" if "plan" in fn_pad else fn_pad
                name_d = "pcnn_conv_wide_plan_create_dilated" if "plan" in fn_dil else fn_dil
                assert _strip(msg_p, name_p) == _strip(msg_d, name_d), (msg_p, msg_d)
            else:
                assert list(a) == list(b)
        if (ph, pw) == (0, 0):
            ok_u, msg_u = _accepts(pkg.conv_wide_plan_info, *base)
            ok_d, msg_d = _accepts(pkg.conv_wide_plan_info, *base, padding=(ph + 1, pw + 1), dilation=(1, 1))
            a, b = (ctypes.c_int * 8)(), (ctypes.c_int * 8)()
            rc_u = L.pcnn_conv_wide_plan_info(*base, W * C, 0, a)
            msg_u = last() if rc_u else ""
            rc_d = L.pcnn_conv_wide_plan_info_dilated(*base, 0, 0, 1, 1, W * C, 0, b)
            msg_d = last() if rc_d else ""
            assert rc_u == rc_d
            if rc_u:
                assert _strip(msg_u, "pcnn_conv_wide_plan_create") == _strip(msg_d, "pcnn_conv_wide_plan_create_dilated")
            else:
                assert list(a) == list(b)
    for N, H, W, C, R, S, st, ph, pw in [(2, 9, 9, 8, 3, 3, 1, 1, 1), (2, 2, 9, 8, 5, 5, 1, 0, 0), (2, 9, 9, 8, 3, 3, 1, 3, 0),
                                         (0, 9, 9, 8, 3, 3, 1, 0, 0), (2, 9, 9, 8, 8, 3, 1, 0, 0), (2, 9, 9, 8, 3, 3, 5, 0, 0)]:
        a, b = (ctypes.c_int * 9)(), (ctypes.c_int * 9)()
        rc_p = L.pcnn_dwconv_info(N, H, W, C, R, S, st, ph, pw, a)
        msg_p = last() if rc_p else ""
        rc_d = L.pcnn_dwconv_info_dilated(N, H, W, C, R, S, st, ph, pw, 1, 1, b)
        msg_d = last() if rc_d else ""
        assert rc_p == rc_d
        if rc_p:
            assert _strip(msg_p, "pcnn_dwconv_info") == _strip(msg_d, "pcnn_dwconv_info_dilated")
        else:
            assert list(a) == list(b)


def test_conv_layer_family_routes_dilated_shapes(pkg):
    """a dilated shape is "wide"; with C % 8 != 0 it is refused (no narrow-channel kernel dilates); a dilated shape the wide plan
    refuses gets that plan's refusal; dilation (1, 1) routes as before"""
    assert pkg.conv_layer_family(2, 14, 14, 32, 32, 3, 3, 1, (2, 2), dilation=(2, 2)) == "wide"
    assert pkg.conv_layer_family(2, 14, 14, 8, 8, 3, 3, 1, (0, 0), dilation=(2, 2)) == "wide"      # narrow at dilation 1
    assert pkg.conv_layer_family(2, 14, 14, 8, 8, 3, 3, 1, (0, 0)) == "narrow"
    assert pkg.conv_layer_family(2, 14, 14, 8, 8, 3, 3, 1, (0, 0), dilation=(1, 1)) == "narrow"
    with pytest.raises(pkg.PcnnError, match="no narrow-channel kernel dilates") as e:
        pkg.conv_layer_family(2, 14, 14, 1, 6, 3, 3, 1, (2, 2), dilation=(2, 2))
    assert e.value.fn == "conv_layer_family"
    with pytest.raises(pkg.PcnnError, match=WIDE_QUERY + ".*K = 264"):
        pkg.conv_layer_family(2, 14, 14, 64, 264, 3, 3, 1, (2, 2), dilation=(2, 2))


# ------------------------------------------------------------------------------------------------- the benchmark's regime
BENCH = [  # N, H, W, C, K, R, S, stride, pad, dilation: `conv_bench.py dilated`
    (128, 56, 56, 64, 64, 3, 3, 1, 1, 1), (128, 56, 56, 64, 64, 3, 3, 1, 2, 2),
    (256, 28, 28, 128, 128, 3, 3, 1, 1, 1), (256, 28, 28, 128, 128, 3, 3, 1, 2, 2), (256, 28, 28, 128, 128, 3, 3, 1, 4, 4),
    (96, 33, 33, 512, 256, 3, 3, 1, 6, 6), (96, 33, 33, 512, 256, 3, 3, 1, 12, 12), (96, 33, 33, 512, 256, 3, 3, 1, 18, 18),
]


def bench_regime(pkg, case, sm):
    N, H, W, C, K, R, S, st, pad, d = case
    fw = pkg.conv_wide_plan_info(N, H, W, C, K, R, S, st, padding=(pad, pad), dilation=(d, d))
    b = pkg.conv_wide_bwd_info(N, H, W, C, K, R, S, st, padding=(pad, pad), dilation=(d, d))
    return dict(fwd=fw["tiles"] // min(fw["tiles"], sm) > 2 * fw["stages"],
                wgrad=b["wgrad_blocks_per_split"] > 2 * b["wgrad_stages"] and b["wgrad_units"] > sm,
                dgrad=b["dgrad_tiles"] // min(b["dgrad_tiles"], sm) > 2 * b["dgrad_stages"],
                groups=b["dgrad_groups"] == (2 if C > 256 else 1), useful=fw["useful_pixels"] == N * H * W)


@pytest.mark.parametrize("case", BENCH, ids=[f"{c[1]}x{c[2]}x{c[3]}-{c[4]}-d{c[9]}" for c in BENCH])
def test_benchmark_shapes_reach_their_regime(pkg, case):
    """at 132 SMs every pass runs more than 2 x stages tiles (or pixel blocks) per CTA, the weight gradient more units than SMs,
    the input gradient two channel groups at C > 256; "same" padding keeps H x W"""
    assert all(bench_regime(pkg, case, 132).values()), bench_regime(pkg, case, 132)
