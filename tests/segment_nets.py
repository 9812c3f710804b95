"""Two segmenters trained on the golden digits (TEST INFRASTRUCTURE ONLY), with the harness shape of example_nets.py: FCNLite (two
transposed convolutions joined to the encoder's skips through batch norm's residual input) and FCNBilinear (a per-pixel head at 7 x 7
and a bilinear resize to 28 x 28).  The targets are segment_ref.digit_masks: 11 classes, 255 ignored."""
import numpy as np
import torch

from example_nets import DEV, Network, nan_buf, same_bits
import segment_ref

O, IGNORE = 11, 255
ENCODER = [("f1", (16, 3, 3, 8), 72), ("f2", (32, 3, 3, 16), 144), ("f3", (64, 3, 3, 32), 288)]


class _Segmenter(Network):
    NB, LR, MOMENTUM, EPOCHS = 32, 0.05, 0.9, 30

    def __init__(self, eng, pkg, p):
        super().__init__(eng)
        B, relu = self.NB, pkg.ACT_RELU
        self.pixels = B * 28 * 28
        self.loss = torch.zeros(self.pixels, dtype=torch.float32, device=DEV)
        self.pred = torch.zeros(self.pixels, dtype=torch.int32, device=DEV)
        self.count = torch.zeros(1, dtype=torch.int32, device=DEV)
        self.c1 = pkg.ConvLayer(eng, B, 28, 28, 8, 16, 3, 3, p["f1"], padding=(1, 1))
        self.c2 = pkg.ConvLayer(eng, B, 28, 28, 16, 32, 3, 3, p["f2"], padding=(1, 1), stride=2)
        self.c3 = pkg.ConvLayer(eng, B, 14, 14, 32, 64, 3, 3, p["f3"], padding=(1, 1), stride=2)
        self.bn1, self.bn2, self.bn3 = (pkg.BatchNormLayer(eng, B, H, H, C, act=relu) for H, C in ((28, 16), (14, 32), (7, 64)))
        self.y1, self.a, self.dy1, self.da = (nan_buf(B, 28, 28, 16) for _ in range(4))
        self.y2, self.b, self.dy2, self.db = (nan_buf(B, 14, 14, 32) for _ in range(4))
        self.y3, self.c, self.dy3, self.dc = (nan_buf(B, 7, 7, 64) for _ in range(4))

    def encode(self, x, training):
        self.c1.forward(x, self.y1)
        self.bn1.forward(self.y1, self.a, training=training)
        self.c2.forward(self.a, self.y2)
        self.bn2.forward(self.y2, self.b, training=training)
        self.c3.forward(self.b, self.y3)
        self.bn3.forward(self.y3, self.c, training=training)

    def encode_backward(self, da_skip=None, db_skip=None):
        self.bn3.backward(self.c, self.dc, self.dy3)
        self.c3.backward(self.y3, self.dy3, self.db)
        self.bn2.backward(self.b, self.db, self.dy2, dy2=db_skip)
        self.c2.backward(self.y2, self.dy2, self.da)
        self.bn1.backward(self.a, self.da, self.dy1, dy2=da_skip)
        self.c1.backward(self.y1, self.dy1, None)

    def pixel_loss(self, z, masks):
        self.eng.softmax_ce_pixels_bf16(z, masks, self.pixels, O, IGNORE, self.dz, self.count, self.loss, self.pred)

    def encoder_layers(self):
        return (self.c1, self.c2, self.c3, self.bn1, self.bn2, self.bn3)


class FCNLite(_Segmenter):
    """conv 16@3x3 pad 1 -> BN+ReLU (a, 28x28) -> conv 32@3x3/2 pad 1 -> BN+ReLU (b, 14x14) -> conv 64@3x3/2 pad 1 -> BN+ReLU (7x7)
    -> ConvTranspose 64->32 4x4/2 pad 1 -> BN + b -> ReLU -> ConvTranspose 32->16 4x4/2 pad 1 -> BN + a -> ReLU -> per-pixel fc 16->11
    -> per-pixel CE (ignore 255).  No conv has a bias."""
    SEED = 31
    PARAMS = ENCODER + [("t1", (64, 32, 4, 4), 64 * 4), ("t2", (32, 16, 4, 4), 32 * 4), ("w", (O, 1, 1, 16), 16), ("bw", O, 16)]

    def __init__(self, eng, pkg, p):
        super().__init__(eng, pkg, p)
        B, relu = self.NB, pkg.ACT_RELU
        self.t1 = pkg.ConvTransposeLayer(eng, B, 7, 7, 64, 32, 4, 4, p["t1"], stride=2, padding=(1, 1))
        self.t2 = pkg.ConvTransposeLayer(eng, B, 14, 14, 32, 16, 4, 4, p["t2"], stride=2, padding=(1, 1))
        self.bn4 = pkg.BatchNormLayer(eng, B, 14, 14, 32, act=relu)
        self.bn5 = pkg.BatchNormLayer(eng, B, 28, 28, 16, act=relu)
        self.fc = pkg.LinearLayer(eng, self.pixels, 1, 1, 16, O, p["w"], p["bw"], row_pitch=16)
        self.y4, self.d, self.dy4, self.dd, self.db_skip = (nan_buf(B, 14, 14, 32) for _ in range(5))
        self.y5, self.e, self.dy5, self.de, self.da_skip = (nan_buf(B, 28, 28, 16) for _ in range(5))
        self.z, self.dz = nan_buf(self.pixels, O), nan_buf(self.pixels, O)

    def forward(self, x, labels, masks, training=True):
        self.encode(x, training)
        self.t1.forward(self.c, self.y4)
        self.bn4.forward(self.y4, self.d, r=self.b, training=training)
        self.t2.forward(self.d, self.y5)
        self.bn5.forward(self.y5, self.e, r=self.a, training=training)
        self.fc.forward(self.e, self.z)
        self.pixel_loss(self.z, masks)

    def backward(self):
        self.fc.backward(self.z, self.dz, self.de)
        self.bn5.backward(self.e, self.de, self.dy5, dr=self.da_skip)
        self.t2.backward(self.y5, self.dy5, self.dd)
        self.bn4.backward(self.d, self.dd, self.dy4, dr=self.db_skip)
        self.t1.backward(self.y4, self.dy4, self.dc)
        self.encode_backward(self.da_skip, self.db_skip)

    def layers(self):
        return (*self.encoder_layers(), self.t1, self.t2, self.bn4, self.bn5, self.fc)


class FCNBilinear(_Segmenter):
    """the same encoder -> per-pixel fc 64->11 at 7x7 -> bilinear 7x7 -> 28x28 -> per-pixel CE (ignore 255)"""
    SEED = 37
    PARAMS = ENCODER + [("w", (O, 1, 1, 64), 64), ("bw", O, 64)]

    def __init__(self, eng, pkg, p):
        super().__init__(eng, pkg, p)
        B = self.NB
        self.fc = pkg.LinearLayer(eng, B * 49, 1, 1, 64, O, p["w"], p["bw"], row_pitch=64)
        self.up = pkg.UpsampleBilinearLayer(eng, B, 7, 7, O, 28, 28)
        self.z7, self.dz7 = nan_buf(B * 49, O), nan_buf(B * 49, O)
        self.z, self.dz = nan_buf(self.pixels, O), nan_buf(self.pixels, O)

    def forward(self, x, labels, masks, training=True):
        self.encode(x, training)
        self.fc.forward(self.c, self.z7)
        self.up.forward(self.z7, self.z)
        self.pixel_loss(self.z, masks)

    def backward(self):
        self.up.backward(self.dz, self.dz7)
        self.fc.backward(self.z7, self.dz7, self.dc)
        self.encode_backward()

    def layers(self):
        return (*self.encoder_layers(), self.fc)

    def stateless(self):
        return (self.up,)


def batchers(eng, pkg, golden, NB):
    """(train, test) ImageBatchers with masks: MNIST at C_out 8, pad-2 crop and flip for training"""
    tr = pkg.ImageBatcher(eng, golden["train_u8"].reshape(-1, 28, 28), golden["train_labels"], NB, pad=2, flip=True, seed=5, C_out=8,
                          masks=segment_ref.digit_masks(golden["train_u8"], golden["train_labels"]))
    te = pkg.ImageBatcher(eng, golden["test_u8"].reshape(-1, 28, 28), golden["test_labels"], NB, shuffle=False, C_out=8,
                          masks=segment_ref.digit_masks(golden["test_u8"], golden["test_labels"]))
    return tr, te


def train_segmenter(eng, pkg, golden, cls, check_step=None):
    """(epoch mean losses, test mIoU, all-background mIoU, params after 5 steps): five checked steps of a fresh network, a second fresh
    network that must match them bit for bit after step 5 and trains for cls.EPOCHS epochs with SGD (momentum), then eval"""
    p = cls.init_params()
    tr, te = batchers(eng, pkg, golden, cls.NB)
    try:
        net = cls(eng, pkg, p)
        opt = pkg.SGD(eng, net.layers(), momentum=cls.MOMENTUM)
        try:
            for it in range(5):
                x, labels, masks = tr.batch(it)
                if check_step:
                    check_step(net, it, x, labels, masks)
                else:
                    net.forward(x, labels, masks)
                    net.backward()
                opt.step(cls.LR)
                eng.sync()
            after5 = net.params()
        finally:
            opt.close()
            net.close()
        net = cls(eng, pkg, p)
        opt = pkg.SGD(eng, net.layers(), momentum=cls.MOMENTUM)
        try:
            losses = []
            for ep in range(cls.EPOCHS):
                tr.epoch = ep
                for s in range(tr.steps_per_epoch):
                    net.forward(*tr.batch(s))
                    net.backward()
                    opt.step(cls.LR)
                    eng.sync()
                    losses.append(float(net.loss.double().sum()) / int(net.count.item()))
                    if ep == 0 and s == 4:
                        eng.sync()
                        assert same_bits(net.params(), after5)
            preds, targets = [], []
            for s in range(te.steps_per_epoch):
                x, labels, masks = te.batch(s, training=False)
                net.forward(x, labels, masks, training=False)
                eng.sync()
                preds.append(net.pred.cpu().numpy())
                targets.append(masks.to_host().reshape(-1))
        finally:
            opt.close()
            net.close()
    finally:
        tr.close()
        te.close()
    spe = len(losses) // cls.EPOCHS
    pred, tgt = np.concatenate(preds), np.concatenate(targets)
    _, _, miou = pkg.segmentation_scores(pred, tgt, O, IGNORE)
    _, _, bg = pkg.segmentation_scores(np.zeros_like(pred), tgt, O, IGNORE)
    return [float(np.mean(losses[e * spe:(e + 1) * spe])) for e in range(cls.EPOCHS)], miou, bg, after5
