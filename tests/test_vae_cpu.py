"""Host-side checks of the variational-autoencoder operations (no GPU): vae_ref's replays of log1p_f32 and sincos_2pi_f32 against
float64 within include/pcnn.h's stated ulp bounds (exhaustively over the Box-Muller inputs), the Philox normals' moments and a
Kolmogorov-Smirnov test, the Gaussian latent and the binary cross-entropy with logits against torch's float64 autograd, and the
domain and partition of pcnn_gaussian_latent_info."""
import numpy as np
import pytest
import scipy.stats
import torch

import vae_ref as V
from restore_ref import bf16_bits, bits_f32

F32 = np.float32
F = torch.nn.functional


def test_log1p_within_its_bound_over_every_box_muller_input():
    k = np.arange(1, 2 ** 24 + 1, dtype=np.int64)
    u1 = k.astype(F32) * V.U24
    got = V.log1p_f32(u1 - F32(1))
    err = V.ulp_error(got, np.log(k.astype(np.float64) * 2.0 ** -24))
    assert err.max() <= V.LOG1P_MAX_ULP, (err.max(), k[np.argmax(err)])
    assert got[-1] == 0 and not np.signbit(got[-1])                         # u1 = 1: radius 0


def test_log1p_within_its_bound_on_zero_to_one():
    rng = np.random.default_rng(7)
    ends = 2.0 ** np.arange(-149, 1)                                         # every binade of [0, 1]: both endpoints
    x = np.unique(np.concatenate([np.linspace(0, 1, 1 << 22).astype(F32), rng.random(1 << 22).astype(F32), ends.astype(F32),
                                  np.nextafter(ends[1:].astype(F32), F32(0)), [F32(0), F32(1)]]))
    err = V.ulp_error(V.log1p_f32(x), np.log1p(x.astype(np.float64)))
    assert err.max() <= V.LOG1P_MAX_ULP, (err.max(), x[np.argmax(err)])


def test_sincos_within_its_bound_over_every_input():
    k = np.arange(1 << 24, dtype=np.int64)
    s, c = V.sincos_2pi_f32(k)
    exact = 2.0 * np.pi * k * 2.0 ** -24
    # float64 sin / cos of the rounded angle miss exact zeros by ~1e-16: take the exact value from the same exact octant reduction
    o, j = k >> 21, k & ((1 << 21) - 1)
    t = np.where(o & 1, (1 << 21) - j, j) * 2.0 ** -21
    S, C = np.sin(np.pi / 4 * t), np.cos(np.pi / 4 * t)
    swap = ((o + 1) >> 1) & 1
    a, b = np.where(swap, C, S), np.where(swap, S, C)
    rs, rc = np.where(o >= 4, -a, a), np.where((o >= 2) & (o <= 5), -b, b)
    assert np.abs(rs - np.sin(exact)).max() < 1e-15 and np.abs(rc - np.cos(exact)).max() < 1e-15
    es, ec = V.ulp_error(s, rs), V.ulp_error(c, rc)
    assert es.max() <= V.SINCOS_MAX_ULP and ec.max() <= V.SINCOS_MAX_ULP, (es.max(), ec.max())


def test_normals_moments_and_ks():
    e = V.eps(1000, 1000, seed=1234, call=1).reshape(-1).astype(np.float64)
    assert e.size == 10 ** 6 and np.all(np.isfinite(e))
    assert abs(e.mean()) < 5e-3 and abs(e.var() - 1) < 5e-3
    assert abs(scipy.stats.skew(e)) < 1e-2 and abs(scipy.stats.kurtosis(e)) < 2e-2
    assert scipy.stats.kstest(e, scipy.stats.norm.cdf).pvalue > 1e-3
    # pairs (2p, 2p + 1) come from one radius: independent coordinates, so uncorrelated
    assert abs(np.corrcoef(e[0::2], e[1::2])[0, 1]) < 5e-3


def test_draws_depend_on_seed_call_and_index_only():
    a = V.eps(7, 12, seed=5, call=3)
    assert np.array_equal(a.reshape(-1)[:60], V.eps(5, 12, seed=5, call=3).reshape(-1))      # a row is (seed, call, r L + j)
    assert not np.array_equal(a, V.eps(7, 12, seed=5, call=4)) and not np.array_equal(a, V.eps(7, 12, seed=6, call=3))


def _stats(rng, R, L, ld, spread=2.0):
    mu = rng.standard_normal((R, L)) * spread
    lv = rng.standard_normal((R, L)) * spread
    s = np.zeros((R, ld), F32)
    s[:, :L], s[:, L:2 * L] = mu, lv
    return bf16_bits(s)


@pytest.mark.parametrize("R,L,ld", [(1, 1, 2), (5, 3, 7), (64, 16, 32), (33, 24, 56), (3, 300, 640)])
def test_latent_is_torchs_float64_autograd(R, L, ld):
    rng = np.random.default_rng(R * 31 + L)
    sb = _stats(rng, R, L, ld)
    seed, call, ks = 99, 2, 0.37
    eps = V.eps(R, L, seed, call).astype(np.float64)
    z, kl = V.latent_fwd(sb, R, L, seed, call, ld=ld)
    s64 = torch.from_numpy(bits_f32(sb).astype(np.float64)).requires_grad_(True)
    mu, lv = s64[:, :L], s64[:, L:2 * L]
    z64 = mu + torch.exp(0.5 * lv) * torch.from_numpy(eps)
    kl64 = 0.5 * (mu * mu + torch.exp(lv) - 1 - lv).sum(1)
    zd = z64.detach().numpy()
    # z: one bf16 rounding of a value within a few fp32 ulps
    assert np.all(np.abs(bits_f32(z) - zd) <= 2 ** -8 * np.abs(zd) + 1e-30)
    assert np.all(np.abs(kl - kl64.detach().numpy()) <= 1e-5 * (0.5 * (mu * mu + torch.exp(lv) + 1 + lv.abs()).sum(1)).detach().numpy())
    zeval, kl2 = V.latent_fwd(sb, R, L, seed, call, ld=ld, training=False)
    assert np.array_equal(zeval, sb.reshape(R, ld)[:, :L]) and np.array_equal(kl2, kl)
    dz = bf16_bits(rng.standard_normal((R, L)).astype(F32))
    ds = V.latent_bwd(sb, dz, R, L, seed, call, ks, ld=ld)
    (z64 * torch.from_numpy(bits_f32(dz).astype(np.float64))).sum().add(ks * kl64.sum()).backward()
    want = s64.grad.numpy()[:, :2 * L]
    got = bits_f32(ds).astype(np.float64)
    scale = np.abs(want) + 2 ** -20 * (np.abs(bits_f32(dz)).max() * np.exp(np.abs(bits_f32(sb)).max()) + ks)
    assert np.all(np.abs(got - want) <= 2 ** -8 * scale)


def test_latent_samples_the_prior_and_keeps_nan():
    R, L = 50, 8
    zero = np.zeros((R, 2 * L), np.uint16)
    z, kl = V.latent_fwd(zero, R, L, seed=3, call=1)
    e = V.eps(R, L, 3, 1)
    assert np.array_equal(z, bf16_bits(e + F32(0))) and np.all(kl == 0)     # bf16(eps), -0 written as +0
    sb = zero.copy()
    sb[0, 0], sb[1, L] = 0x7FC0, 0x7FC0                                      # NaN mu, NaN lv
    z, kl = V.latent_fwd(sb, R, L, seed=3, call=1)
    assert z[0, 0] == 0x7FFF and z[1, 0] == 0x7FFF and np.isnan(kl[0]) and np.isnan(kl[1]) and np.all(kl[2:] == 0)


X_SPECIAL = [0.0, -0.0, 1.0, -1.0, 3.5, -3.5, 17.0, -17.0, 90.0, -90.0, 110.0, -110.0, 1e4, -1e4, 3e38, -3e38]


@pytest.mark.parametrize("t", [0.0, 0.5, 1.0])
def test_bce_is_torchs_float64_autograd(t):
    rng = np.random.default_rng(int(t * 4) + 1)
    x = np.concatenate([X_SPECIAL, rng.standard_normal(2000) * 4, rng.uniform(-1e4, 1e4, 500)]).astype(F32)
    xb = bf16_bits(x)
    tb = bf16_bits(np.full_like(x, t))
    P = x.size
    g, loss = V.bce_replay(xb, tb, 1, 1.0 / P)
    g = g.reshape(-1)
    x64 = torch.from_numpy(bits_f32(xb).astype(np.float64)).requires_grad_(True)
    t64 = torch.full((P,), t, dtype=torch.float64)
    per = F.binary_cross_entropy_with_logits(x64, t64, reduction="none")
    per.mean().backward()
    want = per.detach().numpy()
    # each term: a few fp32 roundings of the term and of x t; torch's own (1 - t) x - logsigmoid(x) cancels to within 2^-52 |x|
    xa = np.abs(bits_f32(xb).astype(np.float64))
    assert np.all(np.abs(loss - want) <= 4 * 2 ** -24 * (np.abs(want) + xa * t) + 2 ** -51 * xa + 1e-37)
    wg = x64.grad.numpy()
    gg = bits_f32(g).astype(np.float64)
    # sigma - t is an fp32 difference (absolute error 2^-24 near sigma = t = 1), then one bf16 rounding (bf16 subnormals: 2^-133)
    assert np.all(np.abs(gg - wg) <= 2 ** -8 * np.abs(wg) + 2 ** -23 / P + 2 ** -133)
    assert np.array_equal(np.signbit(gg[wg == 0]), np.signbit(wg[wg == 0]))


def test_bce_special_values_as_stated():
    x = np.array([np.inf, np.inf, np.inf, -np.inf, -np.inf, -np.inf, np.nan, 1.0], F32)
    t = np.array([0.0, 0.5, 1.0, 0.0, 0.5, 1.0, 0.5, np.nan], F32)
    g, loss = V.bce_replay(bf16_bits(x), bf16_bits(t), 1, 1.0)
    g = g.reshape(-1)
    x64, t64 = torch.from_numpy(x.astype(np.float64)).requires_grad_(True), torch.from_numpy(t.astype(np.float64))
    per = F.binary_cross_entropy_with_logits(x64, t64, reduction="none")
    per.sum().backward()
    gw = x64.grad.numpy()
    # gradients are torch's: 1 - t at +Inf, -t at -Inf, NaN at a NaN operand
    assert np.array_equal(np.isnan(bits_f32(g)), np.isnan(gw)) and np.array_equal(bits_f32(g)[~np.isnan(gw)], gw[~np.isnan(gw)])
    # terms: NaN at +Inf and at (-Inf, t = 0), +Inf at (-Inf, t > 0), NaN at a NaN operand; torch: +Inf at (+Inf, t < 1), else NaN
    assert np.isnan(loss[[0, 1, 2, 3, 6, 7]]).all() and np.all(loss[[4, 5]] == np.inf)
    assert np.all(per.detach().numpy()[[0, 1]] == np.inf) and np.isnan(per.detach().numpy()[[2, 3, 4, 5, 6, 7]]).all()


def test_bce_reads_the_first_c_channels_of_a_pitched_target():
    rng = np.random.default_rng(4)
    xb = bf16_bits(rng.standard_normal((50, 3)).astype(F32) * 3)
    tb = bf16_bits(rng.random((50, 3)).astype(F32))
    wide = rng.integers(0, 0x7F00, (50, 8)).astype(np.uint16)
    wide[:, :3] = tb
    a, la = V.bce_replay(xb, tb, 3, 0.01)
    b, lb = V.bce_replay(xb, wide, 3, 0.01, target_stride=8)
    assert np.array_equal(a, b) and np.array_equal(la, lb)


@pytest.mark.parametrize("R,L,ld,ldz,vec", [(1, 1, 2, 1, 1), (100, 16, 32, 16, 8), (65536, 8, 24, 8, 8), (7, 8, 20, 8, 1),
                                             (9, 8, 16, 12, 1), (3, 4096, 8192, 4096, 8), (130, 5, 10, 5, 1)])
def test_info_partition(pkg, R, L, ld, ldz, vec):
    i = pkg.gaussian_latent_info(R, L, ld, ldz)
    assert i["vec"] == vec and i["threads"] == 256 and i["tile_rows"] == 64 and i["chunk_columns"] % 8 == 0
    assert i["grid"] == -(-R // i["tile_rows"]) and i["smem"] == 4 * i["tile_rows"] * (i["chunk_columns"] + 1)


@pytest.mark.parametrize("R,L,ld,ldz,rule", [(0, 4, 8, 4, "at least 1 row"), (4, 0, 8, 4, "1 <= L <= 4096"),
                                              (4, 4097, 8194, 4097, "1 <= L <= 4096"), (4, 4, 7, 4, "ld >= 2 L"),
                                              (4, 4, 8, 3, "ldz >= L")])
def test_info_refusals(pkg, R, L, ld, ldz, rule):
    with pytest.raises(pkg.PcnnError, match=rule):
        pkg.gaussian_latent_info(R, L, ld, ldz)
    assert pkg.gaussian_latent_info(4, 4)["vec"] == 1 and pkg.gaussian_latent_info(4, 8)["vec"] == 8
