"""A convolutional variational autoencoder trained on the golden digits (TEST INFRASTRUCTURE ONLY), with the harness shape of
restore_nets.py: ConvVAE reads the ImageBatcher's 8-channel batch (channel 0 the digit in [0, 1], the rest zero) and reconstructs
channel 0 as Bernoulli logits, read in place at target_stride 8 by the binary cross-entropy with logits."""
import numpy as np
import torch

from example_nets import DEV, Network, nan_buf, same_bits
from restore_nets import C_IN, batchers, channel0


class ConvVAE(Network):
    """encoder: conv 8->32 3x3/2 pad 1 + ReLU (14 x 14) -> conv 32->64 3x3/2 pad 1 + ReLU (7 x 7) -> fc 3136 -> 2L (mu, logvar);
    latent: GaussianLatentLayer (L = 16); decoder: fc 16 -> 256 + ReLU, read as a dense 4 x 4 x 16 map -> convT 16->32 3x3/2 pad 1 +
    ReLU (7 x 7) -> convT 32->32 3x3/2 pad 1 op 1 + ReLU (14 x 14) -> per-pixel fc 32->4 -> pixel shuffle x2 -> 28 x 28 x 1 logits.
    Loss per image: the sum over its pixels of BCE against channel 0 plus BETA KL, averaged over the batch (BCE scale 1 / B,
    kl_scale BETA / B); AdamW at LR for EPOCHS epochs.  Training draws eps from SEED_LATENT; the test set's from SEED_TEST_LATENT,
    a layer of its own with its own calls, so the test negative ELBO is one fixed Monte-Carlo draw."""
    NB, LR, EPOCHS, L, BETA = 32, 2e-3, 20, 16, 1.0
    SEED = 47
    SEED_LATENT, SEED_TEST_LATENT = 4001, 4002
    PARAMS = [("f1", (32, 3, 3, C_IN), 72), ("b1", 32, 72), ("f2", (64, 3, 3, 32), 288), ("b2", 64, 288),
              ("we", (32, 7, 7, 64), 3136), ("be", 32, 3136), ("wd", (256, 1, 1, 16), 16), ("bd", 256, 16),
              ("t1", (16, 32, 3, 3), 144), ("tb1", 32, 144), ("t2", (32, 32, 3, 3), 288), ("tb2", 32, 288),
              ("w", (4, 1, 1, 32), 32), ("bw", 4, 32)]

    def __init__(self, eng, pkg, p):
        super().__init__(eng)
        B, L, relu = self.NB, self.L, pkg.ACT_RELU
        self.pixels = B * 28 * 28
        self.loss = torch.zeros(self.pixels, dtype=torch.float32, device=DEV)
        self.c1 = pkg.ConvLayer(eng, B, 28, 28, C_IN, 32, 3, 3, p["f1"], p["b1"], act=relu, stride=2, padding=(1, 1))
        self.c2 = pkg.ConvLayer(eng, B, 14, 14, 32, 64, 3, 3, p["f2"], p["b2"], act=relu, stride=2, padding=(1, 1))
        self.enc = pkg.LinearLayer(eng, B, 7, 7, 64, 2 * L, p["we"], p["be"], row_pitch=7 * 64)
        self.lat = pkg.GaussianLatentLayer(eng, B, L, self.SEED_LATENT)
        self.test_lat = pkg.GaussianLatentLayer(eng, B, L, self.SEED_TEST_LATENT)
        self.dec = pkg.LinearLayer(eng, B, 1, 1, L, 256, p["wd"], p["bd"], act=relu, row_pitch=L)
        self.t1 = pkg.ConvTransposeLayer(eng, B, 4, 4, 16, 32, 3, 3, p["t1"], p["tb1"], act=relu, stride=2, padding=(1, 1))
        self.t2 = pkg.ConvTransposeLayer(eng, B, 7, 7, 32, 32, 3, 3, p["t2"], p["tb2"], act=relu, stride=2, padding=(1, 1),
                                         output_padding=(1, 1))
        self.fc = pkg.LinearLayer(eng, B * 196, 1, 1, 32, 4, p["w"], p["bw"], row_pitch=32)
        self.ps = pkg.PixelShuffleLayer(eng, B, 14, 14, 1, 2)
        self.y1, self.dy1 = nan_buf(B, 14, 14, 32), nan_buf(B, 14, 14, 32)
        self.y2, self.dy2 = nan_buf(B, 7, 7, 64), nan_buf(B, 7, 7, 64)
        self.stats, self.z, self.dz = nan_buf(B, 2 * L), nan_buf(B, L), nan_buf(B, L)
        self.h, self.dh = nan_buf(B, 256), nan_buf(B, 256)
        self.a1, self.da1 = nan_buf(B, 7, 7, 32), nan_buf(B, 7, 7, 32)
        self.a2, self.da2 = nan_buf(B, 14, 14, 32), nan_buf(B, 14, 14, 32)
        self.o, self.do = nan_buf(B * 196, 4), nan_buf(B * 196, 4)
        self.out, self.dout = nan_buf(B, 28, 28, 1), nan_buf(B, 28, 28, 1)

    def forward(self, x, training=True):
        """training: eps from the training layer; otherwise from the test layer (a training-mode draw of its own seed)"""
        self.c1.forward(x, self.y1)
        self.c2.forward(self.y1, self.y2)
        self.enc.forward(self.y2, self.stats)
        self.evaluating = not training
        (self.test_lat if self.evaluating else self.lat).forward(self.stats, self.z, training=True)
        self.dec.forward(self.z, self.h)
        self.t1.forward(self.h, self.a1)
        self.t2.forward(self.a1, self.a2)
        self.fc.forward(self.a2, self.o)
        self.ps.forward(self.o, self.out)
        self.eng.bce_logits_loss_bf16(self.out, x, self.pixels, 1, self.dout, self.loss, target_stride=C_IN, scale=1.0 / self.NB)

    def backward(self):
        self.ps.backward(self.dout, self.do)
        self.fc.backward(self.o, self.do, self.da2)
        self.t2.backward(self.a2, self.da2, self.da1)
        self.t1.backward(self.a1, self.da1, self.dh)
        self.dec.backward(self.h, self.dh, self.dz)
        self.lat.backward(self.dz, self.stats, self.BETA / self.NB)          # dstats over stats: enc has no activation
        self.enc.backward(self.stats, self.stats, self.dy2)
        self.c2.backward(self.y2, self.dy2, self.dy1)
        self.c1.backward(self.y1, self.dy1, None)

    def parts(self):
        """(reconstruction, KL) per image of the last forward, float64 [B] each, once the engine's stream has run"""
        rec = self.loss.double().reshape(self.NB, -1).sum(1).cpu().numpy()
        return rec, (self.test_lat if self.evaluating else self.lat).kl.to_host().astype(np.float64)

    def mean_loss(self):
        rec, kl = self.parts()
        return float(np.mean(rec + self.BETA * kl))

    def layers(self):
        return (self.c1, self.c2, self.enc, self.dec, self.t1, self.t2, self.fc)

    def stateless(self):
        return (self.lat, self.test_lat, self.ps)


def mean_image_nelbo(golden, test_x0):
    """the mean-image baseline's negative ELBO per image, in nats: every test image predicted as the training set's per-pixel mean
    of channel 0 (a Bernoulli probability, clipped to [1e-6, 1 - 1e-6] where a pixel is always 0 or 1), KL = 0"""
    tr = golden["train_u8"].reshape(-1, 28, 28)
    mean = np.clip((tr.astype(np.float64) / 255.0).mean(0), 1e-6, 1 - 1e-6)
    t = test_x0.astype(np.float64)
    return float(np.mean(-(t * np.log(mean) + (1 - t) * np.log1p(-mean)).reshape(len(t), -1).sum(1)))


def train_vae(eng, pkg, golden, check_step=None):
    """(epoch mean losses, test negative ELBO, its reconstruction and KL parts, the mean-image baseline, params after 5 steps): five
    checked steps of a fresh network (check_step(net, it, x, the batcher's x array) runs the forward and backward of each), a second
    fresh network that must match them bit for bit after step 5 and trains for EPOCHS epochs with AdamW, then the test digits with
    eps from the test layer.  All per image, in nats."""
    cls = ConvVAE
    p = cls.init_params()
    tr, te = batchers(eng, pkg, golden, cls.NB)
    B = cls.NB
    try:
        net = cls(eng, pkg, p)
        opt = pkg.AdamW(eng, net.layers())
        try:
            for it in range(5):
                x, _ = tr.batch(it)
                if check_step:
                    check_step(net, it, x, tr.x)
                else:
                    net.forward(x)
                    net.backward()
                opt.step(cls.LR)
                eng.sync()
            after5 = net.params()
        finally:
            opt.close()
            net.close()
        net = cls(eng, pkg, p)
        opt = pkg.AdamW(eng, net.layers())
        try:
            losses = []
            for ep in range(cls.EPOCHS):
                tr.epoch = ep
                for s in range(tr.steps_per_epoch):
                    net.forward(tr.batch(s)[0])
                    net.backward()
                    opt.step(cls.LR)
                    eng.sync()
                    losses.append(net.mean_loss())
                    if ep == 0 and s == 4:
                        assert same_bits(net.params(), after5)
            rec, kl, x0 = [], [], []
            for s in range(te.steps_per_epoch):
                x, _ = te.batch(s, training=False)
                net.forward(x, training=False)
                eng.sync()
                r, k = net.parts()
                rec.append(r)
                kl.append(k)
                x0.append(channel0(pkg, te.x.to_host(), B))
        finally:
            opt.close()
            net.close()
    finally:
        tr.close()
        te.close()
    spe = len(losses) // cls.EPOCHS
    rec, kl = float(np.mean(np.concatenate(rec))), float(np.mean(np.concatenate(kl)))
    return ([float(np.mean(losses[e * spe:(e + 1) * spe])) for e in range(cls.EPOCHS)], rec + kl, rec, kl,
            mean_image_nelbo(golden, np.concatenate(x0)), after5)
