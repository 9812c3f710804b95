"""Two image-restoration networks trained on the golden digits (TEST INFRASTRUCTURE ONLY), with the harness shape of
segment_nets.py: ESPCNLite (x2 super-resolution through a pixel shuffle, MSE) and DenoiseNet (masking-noise denoising through a pixel
unshuffle and a pixel shuffle, L1).  Both read the ImageBatcher's 8-channel batch (channel 0 the digit, the rest zero) and
regress channel 0 of the clean high-resolution batch, read in place at target_stride 8."""
import numpy as np
import torch

from example_nets import DEV, Network, nan_buf, same_bits

C_IN = 8                                     # the batcher's C_out: channel 0 is the digit


class _Restorer(Network):
    """What both restorers share: B = 32 images of 28 x 28, a C = 1 prediction out [B][28][28][1] formed by a per-pixel fc to 4
    channels at 14 x 14 and a x2 pixel shuffle, its gradient dout and per-pixel loss, and AdamW at LR for EPOCHS epochs."""
    NB, LR, EPOCHS = 32, 2e-3, 20
    LOSS = None                              # pkg.LOSS_MSE or pkg.LOSS_L1

    def __init__(self, eng, pkg, p, C_fc):
        super().__init__(eng)
        B = self.NB
        self.pixels = B * 28 * 28
        self.loss = torch.zeros(self.pixels, dtype=torch.float32, device=DEV)
        self.fc = pkg.LinearLayer(eng, B * 196, 1, 1, C_fc, 4, p["w"], p["bw"], row_pitch=C_fc)
        self.ps = pkg.PixelShuffleLayer(eng, B, 14, 14, 1, 2)
        self.z, self.dz = nan_buf(B * 196, 4), nan_buf(B * 196, 4)
        self.out, self.dout = nan_buf(B, 28, 28, 1), nan_buf(B, 28, 28, 1)

    def head(self, h, x):
        """fc -> pixel shuffle -> the loss against channel 0 of x, scale 1 / (pixels C)"""
        self.fc.forward(h, self.z)
        self.ps.forward(self.z, self.out)
        self.eng.regression_loss_bf16(self.out, x, self.pixels, 1, self.dout, self.loss, mode=self.LOSS, target_stride=C_IN)

    def head_backward(self, dh):
        self.ps.backward(self.dout, self.dz)
        self.fc.backward(self.z, self.dz, dh)

    def mean_loss(self):
        return float(self.loss.double().sum()) / self.pixels


class ESPCNLite(_Restorer):
    """x2 super-resolution: the 2x2/2 average pool of the batch (14 x 14 x 8, torch's avg_pool2d) -> conv 8->32 5x5 pad 2 + bias + ReLU
    -> conv 32->32 3x3 pad 1 + bias + ReLU -> per-pixel fc 32->4 -> pixel shuffle x2 -> 28 x 28 x 1 -> MSE against the batch's channel
    0.  The baseline is the bilinear x2 of the pooled input."""
    SEED = 41
    PARAMS = [("f1", (32, 5, 5, C_IN), 200), ("b1", 32, 200), ("f2", (32, 3, 3, 32), 288), ("b2", 32, 288), ("w", (4, 1, 1, 32), 32),
              ("bw", 4, 32)]

    def __init__(self, eng, pkg, p):
        super().__init__(eng, pkg, p, 32)
        self.LOSS = pkg.LOSS_MSE
        B, relu = self.NB, pkg.ACT_RELU
        self.pool = pkg.AvgPoolLayer(eng, B, 28, 28, C_IN, 2)
        self.c1 = pkg.ConvLayer(eng, B, 14, 14, C_IN, 32, 5, 5, p["f1"], p["b1"], act=relu, padding=(2, 2))
        self.c2 = pkg.ConvLayer(eng, B, 14, 14, 32, 32, 3, 3, p["f2"], p["b2"], act=relu, padding=(1, 1))
        self.up = pkg.UpsampleBilinearLayer(eng, B, 14, 14, C_IN, 28, 28)
        self.lr, self.bl = nan_buf(B, 14, 14, C_IN), nan_buf(B, 28, 28, C_IN)
        self.y1, self.dy1, self.y2, self.dy2 = (nan_buf(B, 14, 14, 32) for _ in range(4))

    def forward(self, x, training=True):
        self.pool.forward(x, self.lr)
        self.c1.forward(self.lr, self.y1)
        self.c2.forward(self.y1, self.y2)
        self.head(self.y2, x)

    def backward(self):
        self.head_backward(self.dy2)
        self.c2.backward(self.y2, self.dy2, self.dy1)
        self.c1.backward(self.y1, self.dy1, None)

    def baseline(self):
        """[B][28][28][8]: the bilinear x2 of the pooled input of the last forward, once the engine's stream has run"""
        self.up.forward(self.lr, self.bl)
        return self.bl

    def layers(self):
        return (self.c1, self.c2, self.fc)

    def stateless(self):
        return (self.pool, self.up, self.ps)


class DenoiseNet(_Restorer):
    """masking-noise denoising: a DropoutLayer(p = 0.25) corrupts the batch (training forwards draw from SEED_NOISE; the test set's
    from SEED_TEST_NOISE, also in training mode) -> conv 8->16 3x3 pad 1 -> BN+ReLU -> pixel unshuffle x2 (14 x 14 x 64) -> conv
    64->64 3x3 pad 1 -> BN+ReLU -> per-pixel fc 64->4 -> pixel shuffle x2 -> L1 against the clean batch's channel 0.  The convs have no
    bias.  The baseline is the corrupted input itself."""
    SEED = 43
    P_NOISE, SEED_NOISE, SEED_TEST_NOISE = 0.25, 3001, 3002
    PARAMS = [("f1", (16, 3, 3, C_IN), 72), ("f2", (64, 3, 3, 64), 576), ("w", (4, 1, 1, 64), 64), ("bw", 4, 64)]

    def __init__(self, eng, pkg, p):
        super().__init__(eng, pkg, p, 64)
        self.LOSS = pkg.LOSS_L1
        B, relu = self.NB, pkg.ACT_RELU
        self.noise = pkg.DropoutLayer(eng, B, 28 * 28 * C_IN, self.P_NOISE, self.SEED_NOISE)
        self.test_noise = pkg.DropoutLayer(eng, B, 28 * 28 * C_IN, self.P_NOISE, self.SEED_TEST_NOISE)
        self.c1 = pkg.ConvLayer(eng, B, 28, 28, C_IN, 16, 3, 3, p["f1"], None, padding=(1, 1))
        self.c2 = pkg.ConvLayer(eng, B, 14, 14, 64, 64, 3, 3, p["f2"], None, padding=(1, 1))
        self.bn1 = pkg.BatchNormLayer(eng, B, 28, 28, 16, act=relu)
        self.bn2 = pkg.BatchNormLayer(eng, B, 14, 14, 64, act=relu)
        self.un = pkg.PixelUnshuffleLayer(eng, B, 28, 28, 16, 2)
        self.xn = nan_buf(B, 28, 28, C_IN)
        self.y1, self.a, self.da, self.dy1 = (nan_buf(B, 28, 28, 16) for _ in range(4))
        self.u, self.du, self.y2, self.v, self.dv, self.dy2 = (nan_buf(B, 14, 14, 64) for _ in range(6))

    def forward(self, x, training=True):
        (self.noise if training else self.test_noise).forward(x, self.xn, training=True)
        self.c1.forward(self.xn, self.y1)
        self.bn1.forward(self.y1, self.a, training=training)
        self.un.forward(self.a, self.u)
        self.c2.forward(self.u, self.y2)
        self.bn2.forward(self.y2, self.v, training=training)
        self.head(self.v, x)

    def backward(self):
        self.head_backward(self.dv)
        self.bn2.backward(self.v, self.dv, self.dy2)
        self.c2.backward(self.y2, self.dy2, self.du)
        self.un.backward(self.du, self.da)
        self.bn1.backward(self.a, self.da, self.dy1)
        self.c1.backward(self.y1, self.dy1, None)

    def baseline(self):
        """[B][28][28][8]: the corrupted input of the last forward"""
        return self.xn

    def layers(self):
        return (self.c1, self.c2, self.fc, self.bn1, self.bn2)

    def stateless(self):
        return (self.noise, self.test_noise, self.un, self.ps)


def batchers(eng, pkg, golden, NB):
    """(train, test) ImageBatchers: MNIST at C_out 8, pad-2 crop and flip for training, as segment_nets.batchers without masks"""
    tr = pkg.ImageBatcher(eng, golden["train_u8"].reshape(-1, 28, 28), golden["train_labels"], NB, pad=2, flip=True, seed=5, C_out=C_IN)
    te = pkg.ImageBatcher(eng, golden["test_u8"].reshape(-1, 28, 28), golden["test_labels"], NB, shuffle=False, C_out=C_IN)
    return tr, te


def channel0(pkg, bits, B):
    return pkg.bf16_bits_to_f32(np.ascontiguousarray(bits).view(np.uint16)).reshape(B, 28, 28, -1)[..., 0]


def train_restorer(eng, pkg, golden, cls, check_step=None):
    """(epoch mean losses, test PSNR, baseline PSNR, params after 5 steps): five checked steps of a fresh network (check_step(net,
    it, x, the batcher's x array) runs the forward and backward of each), a second fresh
    network that must match them bit for bit after step 5 and trains for cls.EPOCHS epochs with AdamW (lr cls.LR, torch's defaults
    otherwise), then eval on the golden test digits with training=False.  PSNR is pkg.psnr over channel 0 with data range 1."""
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
            preds, base, clean = [], [], []
            for s in range(te.steps_per_epoch):
                x, _ = te.batch(s, training=False)
                net.forward(x, training=False)
                bl = net.baseline()
                eng.sync()
                preds.append(channel0(pkg, net.out.cpu().numpy(), B))
                base.append(channel0(pkg, bl.cpu().numpy(), B))
                clean.append(channel0(pkg, te.x.to_host(), B))
        finally:
            opt.close()
            net.close()
    finally:
        tr.close()
        te.close()
    spe = len(losses) // cls.EPOCHS
    clean = np.concatenate(clean)
    return ([float(np.mean(losses[e * spe:(e + 1) * spe])) for e in range(cls.EPOCHS)], pkg.psnr(np.concatenate(preds), clean),
            pkg.psnr(np.concatenate(base), clean), after5)
