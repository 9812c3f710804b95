"""Variational-autoencoder operations on the H100: the Gaussian latent (pcnn_gaussian_latent_bf16_fwd / _bwd, GaussianLatentLayer)
and the binary cross-entropy with logits (pcnn_bce_logits_bf16) bit for bit against vae_ref.py, canaries in padding columns,
reruns, eval mode, prior sampling, the in-place forms, parity with torch's CUDA autograd, the refusals, and the latent between two
LinearLayers inside SGD and AdamW steps."""
import numpy as np
import pytest
import torch

import vae_ref as V
from example_nets import DEV, host
from restore_ref import bf16_bits, bits_f32

pytestmark = pytest.mark.gpu
NAN = 0x7FC0
F = torch.nn.functional
F32 = np.float32


def dev_bits(bits):
    return torch.from_numpy(np.ascontiguousarray(bits, np.uint16).view(np.int16)).to(DEV)


def stats_bits(rng, R, L, ld, spread=1.5):
    """bf16 stats [R][ld]: mu and lv normal times spread, NaN canaries in the padding columns 2L .. ld-1"""
    s = np.full((R, ld), NAN, np.uint16)
    s[:, :2 * L] = bf16_bits((rng.standard_normal((R, 2 * L)) * spread).astype(F32))
    return s


def canvas(R, ld):
    return torch.full((R * ld + 64,), NAN, dtype=torch.int16, device=DEV)


def rows(buf, R, ld, cols):
    b = host(buf)
    return b[:R * ld].reshape(R, ld)[:, :cols], b[:R * ld].reshape(R, ld)[:, cols:], b[R * ld:]


LATENT = [  # R, L, ld, ldz: both paths, pitched ld and ldz, spatial latents (L = 4, 8 channels of stats per pixel), the benchmark shapes
    (1, 1, 2, 1), (3, 5, 10, 5), (7, 3, 9, 4), (100, 8, 16, 8), (130, 16, 40, 24), (65, 24, 56, 32), (64, 1024, 2048, 1024),
    (5, 1000, 2008, 1000), (2, 4096, 8192, 4096), (1000, 13, 26, 13), (16 * 32 * 32, 4, 8, 4), (65536, 4, 8, 4), (256, 16, 32, 16),
    (65536, 128, 256, 128), (16 * 256 * 256, 4, 8, 4), (8192, 1024, 2048, 1024),
]


@pytest.mark.parametrize("R,L,ld,ldz", LATENT)
def test_latent_bit_exact(pkg, eng, R, L, ld, ldz):
    rng = np.random.default_rng(R * 13 + L)
    sb = stats_bits(rng, R, L, ld)
    seed, call = int(rng.integers(1 << 62)), int(rng.integers(1, 1 << 40))
    stats = dev_bits(sb)
    z, kl = canvas(R, ldz), torch.full((R + 16,), float("nan"), device=DEV)
    eng.gaussian_latent_fwd(stats, z, R, L, seed, call, kl=kl, ld=ld, ldz=ldz)
    eng.sync()
    want_z, want_kl = V.latent_fwd(sb, R, L, seed, call, ld=ld)
    zz, zpad, tail = rows(z, R, ldz, L)
    assert np.array_equal(zz, want_z) and np.all(zpad == NAN) and np.all(tail == NAN)
    kh = kl.cpu().numpy()
    assert np.array_equal(kh[:R].view(np.uint32), want_kl.view(np.uint32)) and np.all(np.isnan(kh[R:]))
    # a rerun gives the same bits; another call other draws
    z2 = canvas(R, ldz)
    eng.gaussian_latent_fwd(stats, z2, R, L, seed, call, ld=ld, ldz=ldz)
    eng.gaussian_latent_fwd(stats, z, R, L, seed, call + 1, kl=kl, ld=ld, ldz=ldz)
    eng.sync()
    assert np.array_equal(rows(z2, R, ldz, L)[0], want_z)
    if R * L >= 16:
        assert not np.array_equal(rows(z, R, ldz, L)[0], want_z)
    # eval: mu's bits, and the same kl
    eng.gaussian_latent_fwd(stats, z, R, L, seed, 0, kl=kl, training=False, ld=ld, ldz=ldz)
    eng.sync()
    assert np.array_equal(rows(z, R, ldz, L)[0], sb[:, :L]) and np.array_equal(kl.cpu().numpy()[:R].view(np.uint32), want_kl.view(np.uint32))
    # backward: dstats with NaN canaries in its padding, then in place over stats
    db = bf16_bits(rng.standard_normal((R, ldz)).astype(F32))
    dz = dev_bits(db)
    ks = float(rng.uniform(0.01, 2.0))
    want = V.latent_bwd(sb, db, R, L, seed, call, ks, ld=ld, ldz=ldz)
    ds = canvas(R, ld)
    eng.gaussian_latent_bwd(stats, dz, ds, R, L, seed, call, ks, ld=ld, ldz=ldz)
    eng.gaussian_latent_bwd(stats, dz, stats, R, L, seed, call, ks, ld=ld, ldz=ldz)
    eng.sync()
    dd, dpad, tail = rows(ds, R, ld, 2 * L)
    assert np.array_equal(dd, want) and np.all(dpad == NAN) and np.all(tail == NAN)
    inplace, ipad, _ = rows(stats, R, ld, 2 * L)
    assert np.array_equal(inplace, want) and np.all(ipad == NAN)


def test_latent_prior_and_in_place_forward(pkg, eng):
    R, L = 4096, 16
    zero = np.zeros((R, 2 * L), np.uint16)
    z = canvas(R, L)
    eng.gaussian_latent_fwd(dev_bits(zero), z, R, L, 11, 1)
    eng.sync()
    assert np.array_equal(rows(z, R, L, L)[0], bf16_bits(V.eps(R, L, 11, 1) + F32(0)))        # bf16(eps), -0 as +0
    rng = np.random.default_rng(2)
    for L, ld in ((16, 32), (5, 12)):
        sb = stats_bits(rng, 300, L, ld)
        stats, kl = dev_bits(sb), torch.zeros(300, device=DEV)
        eng.gaussian_latent_fwd(stats, stats, 300, L, 5, 9, kl=kl, ld=ld, ldz=ld)            # z over mu
        eng.sync()
        want_z, want_kl = V.latent_fwd(sb, 300, L, 5, 9, ld=ld)
        got = host(stats).reshape(300, ld)
        assert np.array_equal(got[:, :L], want_z) and np.array_equal(got[:, L:], sb[:, L:])
        assert np.array_equal(kl.cpu().numpy().view(np.uint32), want_kl.view(np.uint32))


def test_latent_parity_with_torch_cuda_autograd(pkg, eng):
    """torch's float32 CUDA autograd of mu + exp(0.5 lv) eps and 0.5 sum(mu^2 + exp(lv) - 1 - lv), on the same bf16 stats and the
    same eps: z within a bf16 ulp, kl within fp32 summation error, dstats within a bf16 ulp plus the fp32 cancellation of dlv"""
    R, L = 2048, 32
    rng = np.random.default_rng(8)
    sb = stats_bits(rng, R, L, 2 * L)
    db = bf16_bits(rng.standard_normal((R, L)).astype(F32))
    stats, z, kl, ds = dev_bits(sb), canvas(R, L), torch.zeros(R, device=DEV), canvas(R, 2 * L)
    ks = 1.0 / R
    eng.gaussian_latent_fwd(stats, z, R, L, 4, 1, kl=kl)
    eng.gaussian_latent_bwd(stats, dev_bits(db), ds, R, L, 4, 1, ks)
    eng.sync()
    st = torch.from_numpy(bits_f32(sb)).to(DEV).requires_grad_(True)
    eps = torch.from_numpy(V.eps(R, L, 4, 1)).to(DEV)
    mu, lv = st[:, :L], st[:, L:]
    zt = mu + torch.exp(0.5 * lv) * eps
    klt = 0.5 * (mu * mu + torch.exp(lv) - 1 - lv).sum(1)
    g = torch.from_numpy(bits_f32(db)).to(DEV)
    ((zt * g).sum() + ks * klt.sum()).backward()
    # fp32 operations err relative to their operands, so sums that cancel get an absolute allowance of 2^-20 of the operands
    m, s, e, gg = (a.detach().cpu().numpy() for a in (mu, torch.exp(0.5 * lv), eps, g))
    ours_z = bits_f32(rows(z, R, L, L)[0])
    zt = zt.detach().cpu().numpy()
    assert np.all(np.abs(ours_z - zt) <= 2 ** -8 * np.abs(zt) + 2 ** -20 * (np.abs(m) + s * np.abs(e)))
    k = klt.detach().cpu().numpy()
    assert np.all(np.abs(kl.cpu().numpy() - k) <= 1e-5 * (np.abs(k) + L))
    ours_d = bits_f32(rows(ds, R, 2 * L, 2 * L)[0])
    theirs = st.grad.cpu().numpy()
    size = np.concatenate([np.abs(gg) + ks * np.abs(m), np.abs(gg * e) * s + ks * (s * s + 1)], 1)
    assert np.all(np.abs(ours_d - theirs) <= 2 ** -8 * np.abs(theirs) + 2 ** -20 * size)


def bce_operands(rng, P, C, ts, special):
    x = (rng.standard_normal((P, C)) * 4).astype(F32)
    t = rng.random((P, ts)).astype(F32)
    t[:, :C][rng.random((P, C)) < 0.5] = 0.0
    t[:, :C][rng.random((P, C)) < 0.2] = 1.0
    if special:
        xv = [np.inf, -np.inf, np.nan, 0.0, -0.0, 1e4, -1e4, 3e38, 100.0, -120.0, 1.0]
        tv = [0.5, 1.0, 0.5, 0.0, 1.0, 0.0, 1.0, 0.5, 1.0, 0.0, np.nan]
        for k, (a, b) in enumerate(zip(xv, tv)):
            x[k % P, k % C], t[k % P, k % C] = a, b
    return bf16_bits(x), bf16_bits(t)


BCE = [  # pixels, C, target_stride, special: both paths, pitched targets, a C = 80 multi-label head, the benchmark shapes
    (1, 1, 1, False), (1000, 1, 8, True), (4097, 3, 3, True), (300, 3, 7, False), (513, 8, 8, True), (200, 16, 24, True),
    (77, 136, 144, True), (9, 250, 250, True), (4096, 80, 80, True), (128 * 784, 1, 8, False), (16 * 256 * 256, 8, 8, False),
    (65536, 80, 80, False),
]


@pytest.mark.parametrize("P,C,ts,special", BCE)
def test_bce_bit_exact(pkg, eng, P, C, ts, special):
    rng = np.random.default_rng(P + C + ts)
    xb, tb = bce_operands(rng, P, C, ts, special)
    scale = float(rng.uniform(0.1, 2.0)) / (P * C)
    want_g, want_l = V.bce_replay(xb, tb, C, scale, target_stride=ts)
    logits, target = dev_bits(xb), dev_bits(tb)
    d = canvas(P, C)
    loss = torch.full((P + 16,), float("nan"), device=DEV)
    eng.bce_logits_loss_bf16(logits, target, P, C, d, loss, target_stride=ts, scale=scale)
    eng.sync()
    db, lh = host(d), loss.cpu().numpy()
    assert np.all(db[P * C:] == NAN) and np.all(np.isnan(lh[P:]))
    assert np.array_equal(db[:P * C], want_g.reshape(-1))
    nanl = np.isnan(want_l)
    assert np.array_equal(np.isnan(lh[:P]), nanl) and np.array_equal(lh[:P][~nanl].view(np.uint32), want_l[~nanl].view(np.uint32))
    d2 = canvas(P, C)
    eng.bce_logits_loss_bf16(logits, target, P, C, d2, None, target_stride=ts, scale=scale)
    eng.bce_logits_loss_bf16(logits, target, P, C, logits, None, target_stride=ts, scale=scale)         # in place
    eng.sync()
    assert np.array_equal(host(d2)[:P * C], want_g.reshape(-1)) and np.array_equal(host(logits).reshape(-1), want_g.reshape(-1))


def test_bce_default_scale_is_the_mean(pkg, eng):
    rng = np.random.default_rng(3)
    xb, tb = bce_operands(rng, 500, 8, 8, False)
    d = canvas(500, 8)
    eng.bce_logits_loss_bf16(dev_bits(xb), dev_bits(tb), 500, 8, d)
    eng.sync()
    assert np.array_equal(host(d)[:4000], V.bce_replay(xb, tb, 8, 1.0 / 4000)[0].reshape(-1))


def test_bce_parity_with_torch_cuda_autograd(pkg, eng):
    """torch's float32 CUDA binary_cross_entropy_with_logits on the same bf16 logits and targets: dlogits within one bf16 ulp plus
    the fp32 cancellation of sigmoid - t, the mean loss within fp32 summation error"""
    P, C = 20000, 4
    rng = np.random.default_rng(12)
    xb, tb = bce_operands(rng, P, C, C, False)
    d, loss = canvas(P, C), torch.zeros(P, device=DEV)
    eng.bce_logits_loss_bf16(dev_bits(xb), dev_bits(tb), P, C, d, loss)
    eng.sync()
    xt = torch.from_numpy(bits_f32(xb)).to(DEV).reshape(P, C).requires_grad_(True)
    lt = F.binary_cross_entropy_with_logits(xt, torch.from_numpy(bits_f32(tb)).to(DEV).reshape(P, C))
    lt.backward()
    ours, theirs = bits_f32(host(d)[:P * C]).reshape(P, C), xt.grad.cpu().numpy()
    assert np.all(np.abs(ours - theirs) <= 2 ** -8 * np.abs(theirs) + 2 ** -22 / (P * C))
    assert abs(loss.double().sum().item() / (P * C) - lt.item()) <= 1e-5 * lt.item()


def test_refusals(pkg, eng):
    s, z, ds = canvas(64, 32), canvas(64, 16), canvas(64, 32)
    kl = torch.zeros(64, device=DEV)
    base = dict(stats=s, z=z, R=64, L=16, seed=1, call=1, kl=kl, training=True, ld=32, ldz=16)
    for kw, msg in ((dict(R=0), "at least 1 row"), (dict(L=0), "1 <= L <= 4096"), (dict(L=4097, ld=8194, ldz=4097), "1 <= L <= 4096"),
                    (dict(ld=31), "ld >= 2 L"), (dict(ldz=15), "ldz >= L"), (dict(call=0), "call = 0"),
                    (dict(z=z.data_ptr() + 2), "16-byte"), (dict(z=s.data_ptr() + 32), "z overlaps stats"),
                    (dict(z=s, ldz=16), "z overlaps stats"), (dict(kl=s), "kl overlaps"), (dict(stats=None), "NULL")):
        a = dict(base)
        a.update(kw)
        with pytest.raises(pkg.PcnnError, match=msg):
            eng.gaussian_latent_fwd(a["stats"], a["z"], a["R"], a["L"], a["seed"], a["call"], kl=a["kl"], training=a["training"],
                                    ld=a["ld"], ldz=a["ldz"])
    with pytest.raises(pkg.PcnnError, match="training = 2"):
        eng._call("pcnn_gaussian_latent_bf16_fwd", s.data_ptr(), 32, z.data_ptr(), 16, None, 64, 16, 1, 1, 2)
    eng.gaussian_latent_fwd(s, z, 64, 16, 1, 0, training=False, ld=32)                  # eval takes call 0
    for kw, msg in ((dict(call=0), "call = 0"), (dict(kl_scale=float("nan")), "finite kl_scale"), (dict(dstats=s.data_ptr() + 16),
                    "only dstats == stats"), (dict(dz=ds, dstats=ds), "dstats overlaps dz"), (dict(dstats=ds.data_ptr() + 2), "16-byte"),
                    (dict(dz=None), "NULL")):
        a = dict(stats=s, dz=z, dstats=ds, call=1, kl_scale=0.1)
        a.update(kw)
        with pytest.raises(pkg.PcnnError, match=msg):
            eng.gaussian_latent_bwd(a["stats"], a["dz"], a["dstats"], 64, 16, 1, a["call"], a["kl_scale"], ld=32, ldz=16)
    x, y, t = canvas(64, 8), canvas(64, 8), canvas(64, 8)
    loss = torch.zeros(64, device=DEV)
    for kw, msg in ((dict(pixels=0), "pixels = 0"), (dict(C=9, target_stride=8), "target_stride"), (dict(scale=float("inf")), "finite scale"),
                    (dict(dlogits=y.data_ptr() + 2), "16-byte"), (dict(dlogits=x.data_ptr() + 16), "only dlogits == logits"),
                    (dict(dlogits=t), "dlogits overlaps target"), (dict(loss=x), "loss overlaps"), (dict(logits=None), "NULL")):
        a = dict(logits=x, target=t, pixels=64, C=8, dlogits=y, loss=loss, target_stride=8, scale=None)
        a.update(kw)
        with pytest.raises(pkg.PcnnError, match=msg):
            eng.bce_logits_loss_bf16(a["logits"], a["target"], a["pixels"], a["C"], a["dlogits"], a["loss"], a["target_stride"], a["scale"])
    with pytest.raises(pkg.PcnnError, match="mode 2"):                    # the regression loss still refuses mode 2
        eng.regression_loss_bf16(x, t, 64, 8, y, loss, mode=2)


@pytest.mark.parametrize("opt_name", ["SGD", "AdamW"])
def test_latent_between_two_linear_layers(pkg, eng, opt_name):
    """x [N][32] -> fc 32 -> 2L (the encoder) -> latent -> fc L -> 32 (the decoder) -> BCE against x's bits read as probabilities:
    z, kl, dstats and the loss bit for bit against the replays in three steps of the optimizer, the layer's call advancing"""
    N, L, D = 64, 8, 32
    rng = np.random.default_rng(6)
    enc = pkg.LinearLayer(eng, N, 1, 1, D, 2 * L, (rng.standard_normal((2 * L, 1, 1, D)) / 6).astype(F32), np.zeros(2 * L, F32), row_pitch=D)
    dec = pkg.LinearLayer(eng, N, 1, 1, L, D, (rng.standard_normal((D, 1, 1, L)) / 3).astype(F32), np.zeros(D, F32), row_pitch=L)
    lat = pkg.GaussianLatentLayer(eng, N, L, seed=77)
    opt = pkg.SGD(eng, [enc, dec], momentum=0.9) if opt_name == "SGD" else pkg.AdamW(eng, [enc, dec])
    xb = bf16_bits(rng.random((N, D)).astype(F32))
    x = dev_bits(xb)
    stats, z, y, dy, dz, dx = canvas(N, 2 * L), canvas(N, L), canvas(N, D), canvas(N, D), canvas(N, L), canvas(N, D)
    loss = torch.zeros(N, device=DEV)
    beta = 0.5
    totals = []
    try:
        for step in range(3):
            enc.forward(x, stats)
            lat.forward(stats, z)
            dec.forward(z, y)
            eng.bce_logits_loss_bf16(y, x, N, D, dy, loss, scale=1.0 / N)
            eng.sync()
            sb = host(stats)[:N * 2 * L].copy()
            want_z, want_kl = V.latent_fwd(sb, N, L, 77, step + 1)
            assert lat.call == step + 1 and np.array_equal(host(z)[:N * L].reshape(N, L), want_z)
            assert np.array_equal(lat.kl.to_host().view(np.uint32), want_kl.view(np.uint32))
            g, lw = V.bce_replay(host(y)[:N * D], xb, D, 1.0 / N)
            assert np.array_equal(host(dy)[:N * D], g.reshape(-1)) and np.array_equal(loss.cpu().numpy().view(np.uint32), lw.view(np.uint32))
            dec.backward(y, dy, dz)
            lat.backward(dz, stats, beta / N)                               # dstats in place over stats
            enc.backward(stats, stats, dx)
            eng.sync()
            want = V.latent_bwd(sb, host(dz)[:N * L], N, L, 77, step + 1, beta / N)
            assert np.array_equal(host(stats)[:N * 2 * L].reshape(N, 2 * L), want)
            totals.append(float(lw.astype(np.float64).sum() + beta * want_kl.astype(np.float64).sum()) / N)
            opt.step(0.05 if opt_name == "SGD" else 0.01)
        assert np.all(np.isfinite(totals)) and totals[2] < totals[0]
        lat.forward(stats, z, training=False)
        assert lat.call == 3
    finally:
        opt.close()
        for layer in (enc, dec, lat):
            layer.close()
