"""The example networks that the end-to-end tests train on the golden MNIST subset, and the one loop that trains them (TEST
INFRASTRUCTURE ONLY).

Each network is a class over the device-trained layers of the package passed to it, with its batch size NB, its step LR_STEP, its
EPOCHS and its fan-scaled uniform initialisation as class attributes.  The per-layer checks and the accuracy thresholds stay in the
tests that own them; the float32 torch CPU replicas under scripts/ take the hyperparameters and initial masters from here.

train() is the end-to-end schedule every such test runs: five checked steps of a fresh network, a second fresh network that must
reach the first's parameters bit for bit after step 5 and then trains for its epochs, and eval with training=False."""
import numpy as np
import torch

DEV = torch.device("cuda", 0)
NAN_BF16 = 0x7FC0
ROW_BYTES = 28 * 32 * 2              # one image of mnist_device: 28 rows of 32 bf16


def nan_buf(*shape):
    return torch.full(shape, NAN_BF16, dtype=torch.int16, device=DEV)


def host(t):
    return t.cpu().numpy().view(np.uint16)


def mnist_device(pkg, u8):
    """uint8 digits [n][28][28] as bf16 [n * 28][32] on the device: x / 255, two zero columns per row"""
    n = u8.shape[0]
    xl = np.zeros((n * 28, 32), np.uint16)
    xl[:, :28] = pkg.f32_to_bf16_bits(u8.reshape(n, 28, 28).astype(np.float32) / 255.0).reshape(n * 28, 28)
    return torch.from_numpy(xl.view(np.int16)).to(DEV)


class Slices:
    """golden digits in mnist_device's layout, NB per step in order: the interface of pkg.ImageBatcher (batch, steps_per_epoch,
    epoch) without a shuffle or augmentation"""

    def __init__(self, pkg, u8, labels, NB):
        self.x, self.labels, self.NB = mnist_device(pkg, u8), torch.from_numpy(labels).to(DEV), NB
        self.steps_per_epoch = len(labels) // NB
        self.epoch = 0

    def batch(self, s, training=True):
        """(pointer to the first image, labels) of slice s"""
        return self.x.data_ptr() + s * self.NB * ROW_BYTES, self.labels[s * self.NB:(s + 1) * self.NB]


def fan_uniform(seed, spec):
    """{name: U(-1, 1) / sqrt(fan) as float32} for (name, shape, fan) in spec, drawn in that order from one generator"""
    rng = np.random.default_rng(seed)
    return {name: rng.uniform(-1, 1, shape).astype(np.float32) / np.float32(np.sqrt(fan)) for name, shape, fan in spec}


def same_bits(a, b):
    return len(a) == len(b) and all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(a, b))


class Network:
    """What every example network shares: the engine, the loss and pred of its softmax cross-entropy, and sgd, params and close
    over its layers.  layers() lists the trained layers (the optimizers take them), stateless() the parameter-free ones.  They are
    methods, not lists held by the instance, so that each layer is reachable through one attribute only: network_tape.layers_of
    walks vars(net) and would wrap a layer twice."""
    NB, LR_STEP, EPOCHS = 128, None, None
    SEED, PARAMS = None, ()                     # fan_uniform's seed and (name, shape, fan) list of the masters

    def __init__(self, eng):
        self.eng = eng
        self.loss = torch.zeros(self.NB, dtype=torch.float32, device=DEV)
        self.pred = torch.zeros(self.NB, dtype=torch.int32, device=DEV)

    @classmethod
    def init_params(cls):
        return fan_uniform(cls.SEED, cls.PARAMS)

    def layers(self):
        raise NotImplementedError

    def stateless(self):
        return ()

    def sgd(self, lr):
        for layer in self.layers():
            layer.sgd(lr)

    def params(self):
        return [a for layer in self.layers() for a in layer.params() if a is not None]

    def close(self):
        for layer in (*self.layers(), *self.stateless()):
            layer.close()


LENET_PARAMS = [("f1", (8, 5, 5, 1), 25), ("b1", 8, 25), ("f2", (16, 3, 3, 8), 72), ("b2", 16, 72), ("w3", (128, 6, 6, 16), 576),
                ("b3", 128, 576), ("w4", (10, 1, 1, 128), 128), ("b4", 10, 128)]


class Net(Network):
    """conv 8@5x5 sigmoid -> pool 2 -> conv 16@3x3 pad 1 -> pool 2 -> fc 576->128 sigmoid -> fc 128->10 -> softmax CE (1/B)"""
    LR_STEP, EPOCHS = 0.3, 40
    SEED, PARAMS = 5, LENET_PARAMS

    def __init__(self, eng, pkg, p):
        super().__init__(eng)
        B = self.NB
        self.c1 = pkg.ConvLayer(eng, B, 28, 28, 1, 8, 5, 5, p["f1"], p["b1"], act=1)
        self.c2 = pkg.ConvLayer(eng, B, 12, 12, 8, 16, 3, 3, p["f2"], p["b2"], act=0, padding=(1, 1))
        self.fc1 = pkg.LinearLayer(eng, B, 6, 6, 16, 128, p["w3"], p["b3"], act=1)
        self.fc2 = pkg.LinearLayer(eng, B, 1, 1, 128, 10, p["w4"], p["b4"], act=0, row_pitch=128)
        self.p1 = pkg.MaxPoolLayer(eng, B, 24, 24, 8, 2, row_pitch=self.c2.row_pitch, image_rows=self.c2.image_rows)
        self.p2 = pkg.MaxPoolLayer(eng, B, 12, 12, 16, 2, row_pitch=self.fc1.row_pitch, image_rows=self.fc1.image_rows)
        self.y1, self.dy1 = nan_buf(B, 24, 24, 8), nan_buf(B, 24, 24, 8)
        self.x2, self.dx2 = nan_buf(B, 12, self.c2.row_pitch), nan_buf(B, 12, self.c2.row_pitch)
        self.y2, self.dy2 = nan_buf(B, 12, 12, 16), nan_buf(B, 12, 12, 16)
        self.x3, self.dx3 = nan_buf(B, 6, 96), nan_buf(B, 6, 96)
        self.y3, self.dy3 = nan_buf(B, 128), nan_buf(B, 128)
        self.z, self.dz = nan_buf(B, 10), nan_buf(B, 10)

    def forward(self, x, labels, training=True):
        """training changes nothing: the network has no batch statistics and no dropout"""
        B = self.NB
        self.c1.forward(x, self.y1)
        self.p1.forward(self.y1, self.x2)
        self.c2.forward(self.x2, self.y2)
        self.p2.forward(self.y2, self.x3)
        self.fc1.forward(self.x3, self.y3)
        self.fc2.forward(self.y3, self.z)
        self.eng.softmax_ce_bf16(self.z, labels, B, 10, 1.0 / B, self.dz, self.loss, self.pred)

    def backward(self, hook=lambda name: None):
        self.fc2.backward(self.z, self.dz, self.dy3)
        hook("fc2")
        self.fc1.backward(self.y3, self.dy3, self.dx3)
        hook("fc1")
        self.p2.backward(self.dx3, self.dy2)
        self.c2.backward(self.y2, self.dy2, self.dx2)
        self.p1.backward(self.dx2, self.dy1)
        self.c1.backward(self.y1, self.dy1, None)

    def layers(self):
        return (self.c1, self.c2, self.fc1, self.fc2)

    def stateless(self):
        return (self.p1, self.p2)


class ReluNet(Network):
    """conv 8@5x5 ReLU -> pool 2 -> conv 16@3x3 pad 1 ReLU -> pool 2 -> fc 576->128 ReLU -> fc 128->10 -> softmax CE (1/B)"""
    LR_STEP, EPOCHS = 0.05, 40
    SEED, PARAMS = 5, LENET_PARAMS

    def __init__(self, eng, pkg, p):
        super().__init__(eng)
        B = self.NB
        relu = pkg.ACT_RELU
        self.c1 = pkg.ConvLayer(eng, B, 28, 28, 1, 8, 5, 5, p["f1"], p["b1"], act=relu)
        self.c2 = pkg.ConvLayer(eng, B, 12, 12, 8, 16, 3, 3, p["f2"], p["b2"], act=relu, padding=(1, 1))
        self.fc1 = pkg.LinearLayer(eng, B, 6, 6, 16, 128, p["w3"], p["b3"], act=relu)
        self.fc2 = pkg.LinearLayer(eng, B, 1, 1, 128, 10, p["w4"], p["b4"], act=pkg.ACT_NONE, row_pitch=128)
        self.p1 = pkg.MaxPoolLayer(eng, B, 24, 24, 8, 2, row_pitch=self.c2.row_pitch, image_rows=self.c2.image_rows)
        self.p2 = pkg.MaxPoolLayer(eng, B, 12, 12, 16, 2, row_pitch=self.fc1.row_pitch, image_rows=self.fc1.image_rows)
        self.y1, self.dy1 = nan_buf(B, 24, 24, 8), nan_buf(B, 24, 24, 8)
        self.x2, self.dx2 = nan_buf(B, 12, self.c2.row_pitch), nan_buf(B, 12, self.c2.row_pitch)
        self.y2, self.dy2 = nan_buf(B, 12, 12, 16), nan_buf(B, 12, 12, 16)
        self.x3, self.dx3 = nan_buf(B, 6, 96), nan_buf(B, 6, 96)
        self.y3, self.dy3 = nan_buf(B, 128), nan_buf(B, 128)
        self.z, self.dz = nan_buf(B, 10), nan_buf(B, 10)

    def forward(self, x, labels, training=True):
        """training changes nothing: the network has no batch statistics and no dropout"""
        B = self.NB
        self.c1.forward(x, self.y1)
        self.p1.forward(self.y1, self.x2)
        self.c2.forward(self.x2, self.y2)
        self.p2.forward(self.y2, self.x3)
        self.fc1.forward(self.x3, self.y3)
        self.fc2.forward(self.y3, self.z)
        self.eng.softmax_ce_bf16(self.z, labels, B, 10, 1.0 / B, self.dz, self.loss, self.pred)

    def backward(self, hook=lambda name, y, dy: None):
        """hook(name, y, dy) runs before and after each ReLU layer's backward, which rewrites dy in place"""
        self.fc2.backward(self.z, self.dz, self.dy3)
        for name, layer, y, dy, dx, pool in (("fc1", self.fc1, self.y3, self.dy3, self.dx3, None),
                                             ("c2", self.c2, self.y2, self.dy2, self.dx2, (self.p2, self.dx3)),
                                             ("c1", self.c1, self.y1, self.dy1, None, (self.p1, self.dx2))):
            if pool is not None:
                pool[0].backward(pool[1], dy)
            hook(name + ":before", y, dy)
            layer.backward(y, dy, dx)
            hook(name + ":after", y, dy)

    def layers(self):
        return (self.c1, self.c2, self.fc1, self.fc2)

    def stateless(self):
        return (self.p1, self.p2)


class ResNet(Network):
    """conv 8@5x5 -> BN+ReLU -> pool 2 -> conv 16@3x3 pad 1 -> BN+ReLU (x0) -> [conv 16@3x3 pad 1 -> BN+ReLU -> conv 16@3x3 pad 1
    -> BN + x0 -> ReLU] -> pool 2 -> fc 576->10 -> softmax CE (1/B).  The convs have no bias."""
    LR_STEP, EPOCHS = 0.05, 40
    SEED, PARAMS = 7, [("f1", (8, 5, 5, 1), 25), ("f2", (16, 3, 3, 8), 72), ("f3", (16, 3, 3, 16), 144), ("f4", (16, 3, 3, 16), 144),
                       ("w5", (10, 6, 6, 16), 576), ("b5", 10, 576)]

    def __init__(self, eng, pkg, p):
        super().__init__(eng)
        relu, none = pkg.ACT_RELU, pkg.ACT_NONE
        B = self.NB
        self.c1 = pkg.ConvLayer(eng, B, 28, 28, 1, 8, 5, 5, p["f1"], None, act=none)
        self.c2 = pkg.ConvLayer(eng, B, 12, 12, 8, 16, 3, 3, p["f2"], None, act=none, padding=(1, 1))
        self.c3 = pkg.ConvLayer(eng, B, 12, 12, 16, 16, 3, 3, p["f3"], None, act=none, padding=(1, 1))
        self.c4 = pkg.ConvLayer(eng, B, 12, 12, 16, 16, 3, 3, p["f4"], None, act=none, padding=(1, 1))
        assert self.c3.row_pitch == 12 * 16 and self.c4.row_pitch == 12 * 16     # a dense BN output is their x layout
        self.fc = pkg.LinearLayer(eng, B, 6, 6, 16, 10, p["w5"], p["b5"], act=none)
        self.bn = [pkg.BatchNormLayer(eng, B, 24, 24, 8, act=relu)] + [pkg.BatchNormLayer(eng, B, 12, 12, 16, act=relu) for _ in range(3)]
        self.p1 = pkg.MaxPoolLayer(eng, B, 24, 24, 8, 2, row_pitch=self.c2.row_pitch, image_rows=self.c2.image_rows)
        self.p2 = pkg.MaxPoolLayer(eng, B, 12, 12, 16, 2, row_pitch=self.fc.row_pitch, image_rows=self.fc.image_rows)
        self.y1, self.z1, self.dz1, self.dy1 = (nan_buf(B, 24, 24, 8) for _ in range(4))
        self.x2, self.dx2 = nan_buf(B, 12, self.c2.row_pitch), nan_buf(B, 12, self.c2.row_pitch)
        (self.y2, self.x0, self.y3, self.z3, self.y4, self.out, self.dout, self.dy4, self.dres, self.dz3, self.dy3, self.dx0,
         self.dy2) = (nan_buf(B, 12, 12, 16) for _ in range(13))
        self.x5, self.dx5 = nan_buf(B, 6, self.fc.row_pitch), nan_buf(B, 6, self.fc.row_pitch)
        self.z, self.dz = nan_buf(B, 10), nan_buf(B, 10)

    def forward(self, x, labels, training=True):
        b1, b2, b3, b4 = self.bn
        self.c1.forward(x, self.y1)
        b1.forward(self.y1, self.z1, training=training)
        self.p1.forward(self.z1, self.x2)
        self.c2.forward(self.x2, self.y2)
        b2.forward(self.y2, self.x0, training=training)
        self.c3.forward(self.x0, self.y3)
        b3.forward(self.y3, self.z3, training=training)
        self.c4.forward(self.z3, self.y4)
        b4.forward(self.y4, self.out, r=self.x0, training=training)
        self.p2.forward(self.out, self.x5)
        self.fc.forward(self.x5, self.z)
        self.eng.softmax_ce_bf16(self.z, labels, self.NB, 10, 1.0 / self.NB, self.dz, self.loss, self.pred)

    def backward(self):
        b1, b2, b3, b4 = self.bn
        self.fc.backward(self.z, self.dz, self.dx5)
        self.p2.backward(self.dx5, self.dout)
        b4.backward(self.out, self.dout, self.dy4, dr=self.dres)
        self.c4.backward(self.y4, self.dy4, self.dz3)
        b3.backward(self.z3, self.dz3, self.dy3)
        self.c3.backward(self.y3, self.dy3, self.dx0)
        b2.backward(self.x0, self.dx0, self.dy2, dy2=self.dres)
        self.c2.backward(self.y2, self.dy2, self.dx2)
        self.p1.backward(self.dx2, self.dz1)
        b1.backward(self.z1, self.dz1, self.dy1)
        self.c1.backward(self.y1, self.dy1, None)

    # (BN layer, its x, r, y, dy, dy2, dx) for the replays
    def bn_tensors(self):
        b1, b2, b3, b4 = self.bn
        return [(b1, self.y1, None, self.z1, self.dz1, None, self.dy1), (b2, self.y2, None, self.x0, self.dx0, self.dres, self.dy2),
                (b3, self.y3, None, self.z3, self.dz3, None, self.dy3), (b4, self.y4, self.x0, self.out, self.dout, None, self.dy4)]

    def layers(self):
        return (self.c1, self.c2, self.c3, self.c4, self.fc, *self.bn)

    def stateless(self):
        return (self.p1, self.p2)


class ResNetGAP(Network):
    """conv 8@5x5 -> BN+ReLU -> avg pool 2 -> conv 16@3x3 pad 1 -> BN+ReLU (x0) -> [conv 16@3x3 pad 1 -> BN+ReLU -> conv 16@3x3
    pad 1 -> BN + x0 -> ReLU] (x1) -> [conv 32@3x3 stride 2 pad 1 -> BN+ReLU -> conv 32@3x3 pad 1 -> BN + s -> ReLU, s = BN(conv
    32@3x3 stride 2 pad 1 (x1))] -> GAP -> fc 32->10 -> softmax CE (1/B).  The convs have no bias.  The projection is 3x3 rather
    than ResNet's 1x1: a 1x1 stride-2 conv over 16 channels is a row-Toeplitz layer, whose input gradient has no 1x1 kernel."""
    LR_STEP, EPOCHS = 0.2, 40
    SEED, PARAMS = 9, [("f1", (8, 5, 5, 1), 25), ("f2", (16, 3, 3, 8), 72), ("f3", (16, 3, 3, 16), 144), ("f4", (16, 3, 3, 16), 144),
                       ("f5", (32, 3, 3, 16), 144), ("f6", (32, 3, 3, 32), 288), ("f7", (32, 3, 3, 16), 144), ("w8", (10, 1, 1, 32), 32),
                       ("b8", 10, 32)]

    def __init__(self, eng, pkg, p):
        super().__init__(eng)
        relu, none = pkg.ACT_RELU, pkg.ACT_NONE
        B = self.NB
        conv = lambda H, C, K, R, f, **k: pkg.ConvLayer(eng, B, H, H, C, K, R, R, p[f], None, act=none, **k)
        self.c1 = conv(28, 1, 8, 5, "f1")
        self.c2 = conv(12, 8, 16, 3, "f2", padding=(1, 1))
        self.c3, self.c4 = conv(12, 16, 16, 3, "f3", padding=(1, 1)), conv(12, 16, 16, 3, "f4", padding=(1, 1))
        self.c5 = conv(12, 16, 32, 3, "f5", padding=(1, 1), stride=2)
        self.c6 = conv(6, 32, 32, 3, "f6", padding=(1, 1))
        self.c7 = conv(12, 16, 32, 3, "f7", padding=(1, 1), stride=2)
        assert self.c5.out_shape == self.c7.out_shape == (B, 6, 6, 32)
        BN = lambda H, C, act: pkg.BatchNormLayer(eng, B, H, H, C, act=act)
        self.bn = [BN(24, 8, relu), BN(12, 16, relu), BN(12, 16, relu), BN(12, 16, relu), BN(6, 32, relu), BN(6, 32, relu), BN(6, 32, none)]
        self.pool = pkg.AvgPoolLayer(eng, B, 24, 24, 8, 2, row_pitch=self.c2.row_pitch, image_rows=self.c2.image_rows)
        self.gap = pkg.GlobalAvgPoolLayer(eng, B, 6, 6, 32)
        self.fc = pkg.LinearLayer(eng, B, 1, 1, 32, 10, p["w8"], p["b8"], act=none, row_pitch=self.gap.row_pitch)
        self.y1, self.z1, self.dz1, self.dy1 = (nan_buf(B, 24, 24, 8) for _ in range(4))
        self.x2, self.dx2 = nan_buf(B, 12, self.c2.row_pitch), nan_buf(B, 12, self.c2.row_pitch)
        (self.y2, self.x0, self.y3, self.z3, self.y4, self.x1, self.dx1, self.dx1p, self.dy4, self.dres, self.dz3, self.dy3, self.dx0,
         self.dy2) = (nan_buf(B, 12, 12, 16) for _ in range(14))
        (self.y5, self.z5, self.y6, self.out, self.y7, self.s, self.dout, self.dy6, self.ds, self.dy7, self.dz5,
         self.dy5) = (nan_buf(B, 6, 6, 32) for _ in range(12))
        self.h, self.dh = nan_buf(B, self.gap.row_pitch), nan_buf(B, self.gap.row_pitch)
        self.z, self.dz = nan_buf(B, 10), nan_buf(B, 10)

    def forward(self, x, labels, training=True):
        b1, b2, b3, b4, b5, b6, b7 = self.bn
        self.c1.forward(x, self.y1)
        b1.forward(self.y1, self.z1, training=training)
        self.pool.forward(self.z1, self.x2)
        self.c2.forward(self.x2, self.y2)
        b2.forward(self.y2, self.x0, training=training)
        self.c3.forward(self.x0, self.y3)
        b3.forward(self.y3, self.z3, training=training)
        self.c4.forward(self.z3, self.y4)
        b4.forward(self.y4, self.x1, r=self.x0, training=training)
        self.c5.forward(self.x1, self.y5)
        b5.forward(self.y5, self.z5, training=training)
        self.c6.forward(self.z5, self.y6)
        self.c7.forward(self.x1, self.y7)
        b7.forward(self.y7, self.s, training=training)
        b6.forward(self.y6, self.out, r=self.s, training=training)
        self.gap.forward(self.out, self.h)
        self.fc.forward(self.h, self.z)
        self.eng.softmax_ce_bf16(self.z, labels, self.NB, 10, 1.0 / self.NB, self.dz, self.loss, self.pred)

    def backward(self):
        b1, b2, b3, b4, b5, b6, b7 = self.bn
        self.fc.backward(self.z, self.dz, self.dh)
        self.gap.backward(self.dh, self.dout)
        b6.backward(self.out, self.dout, self.dy6, dr=self.ds)
        self.c6.backward(self.y6, self.dy6, self.dz5)
        b5.backward(self.z5, self.dz5, self.dy5)
        self.c5.backward(self.y5, self.dy5, self.dx1)
        b7.backward(self.s, self.ds, self.dy7)
        self.c7.backward(self.y7, self.dy7, self.dx1p)
        b4.backward(self.x1, self.dx1, self.dy4, dr=self.dres, dy2=self.dx1p)      # main path and projection meet at x1
        self.c4.backward(self.y4, self.dy4, self.dz3)
        b3.backward(self.z3, self.dz3, self.dy3)
        self.c3.backward(self.y3, self.dy3, self.dx0)
        b2.backward(self.x0, self.dx0, self.dy2, dy2=self.dres)
        self.c2.backward(self.y2, self.dy2, self.dx2)
        self.pool.backward(self.dx2, self.dz1)
        b1.backward(self.z1, self.dz1, self.dy1)
        self.c1.backward(self.y1, self.dy1, None)

    def layers(self):
        return (self.c1, self.c2, self.c3, self.c4, self.c5, self.c6, self.c7, self.fc, *self.bn)

    def stateless(self):
        return (self.pool, self.gap)


class SEResNet(ResNetGAP):
    """The GAP ResNet with squeeze-and-excitation in both residual blocks: each block's last BN runs without r and ReLU, and an SE
    layer (16 -> 8 -> 16, then 32 -> 8 -> 32) carries the residual add and the ReLU.  The GAP ResNet's masters, then the SE
    layers' (fc1 w, b, fc2 w, b of each) from a second generator."""
    SE_SEED, SE_PARAMS = 10, [(f"{k}_{n}", shape, fan) for k, C in (("se1", 16), ("se2", 32))
                              for n, shape, fan in (("w1", (8, C), C), ("b1", 8, C), ("w2", (C, 8), 8), ("b2", C, 8))]

    @classmethod
    def init_params(cls):
        return {**super().init_params(), **fan_uniform(cls.SE_SEED, cls.SE_PARAMS)}

    def __init__(self, eng, pkg, p):
        Network.__init__(self, eng)
        relu, none = pkg.ACT_RELU, pkg.ACT_NONE
        B = self.NB
        conv = lambda H, C, K, R, f, **k: pkg.ConvLayer(eng, B, H, H, C, K, R, R, p[f], None, act=none, **k)
        self.c1 = conv(28, 1, 8, 5, "f1")
        self.c2 = conv(12, 8, 16, 3, "f2", padding=(1, 1))
        self.c3, self.c4 = conv(12, 16, 16, 3, "f3", padding=(1, 1)), conv(12, 16, 16, 3, "f4", padding=(1, 1))
        self.c5 = conv(12, 16, 32, 3, "f5", padding=(1, 1), stride=2)
        self.c6 = conv(6, 32, 32, 3, "f6", padding=(1, 1))
        self.c7 = conv(12, 16, 32, 3, "f7", padding=(1, 1), stride=2)
        BN = lambda H, C, act: pkg.BatchNormLayer(eng, B, H, H, C, act=act)
        self.bn = [BN(24, 8, relu), BN(12, 16, relu), BN(12, 16, relu), BN(12, 16, none), BN(6, 32, relu), BN(6, 32, none), BN(6, 32, none)]
        se = lambda k: [p[f"{k}_{n}"] for n in ("w1", "b1", "w2", "b2")]
        self.se1 = pkg.SqueezeExcitationLayer(eng, B, 12, 12, 16, 8, *se("se1"), act=relu)
        self.se2 = pkg.SqueezeExcitationLayer(eng, B, 6, 6, 32, 8, *se("se2"), act=relu)
        self.pool = pkg.AvgPoolLayer(eng, B, 24, 24, 8, 2, row_pitch=self.c2.row_pitch, image_rows=self.c2.image_rows)
        self.gap = pkg.GlobalAvgPoolLayer(eng, B, 6, 6, 32)
        self.fc = pkg.LinearLayer(eng, B, 1, 1, 32, 10, p["w8"], p["b8"], act=none, row_pitch=self.gap.row_pitch)
        self.y1, self.z1, self.dz1, self.dy1 = (nan_buf(B, 24, 24, 8) for _ in range(4))
        self.x2, self.dx2 = nan_buf(B, 12, self.c2.row_pitch), nan_buf(B, 12, self.c2.row_pitch)
        (self.y2, self.x0, self.y3, self.z3, self.y4, self.z4, self.x1, self.dx1, self.dx1p, self.dz4, self.dy4, self.dres, self.dz3,
         self.dy3, self.dx0, self.dy2) = (nan_buf(B, 12, 12, 16) for _ in range(16))
        (self.y5, self.z5, self.y6, self.z6, self.out, self.y7, self.s, self.dout, self.dz6, self.dy6, self.ds, self.dy7, self.dz5,
         self.dy5) = (nan_buf(B, 6, 6, 32) for _ in range(14))
        self.h, self.dh = nan_buf(B, self.gap.row_pitch), nan_buf(B, self.gap.row_pitch)
        self.z, self.dz = nan_buf(B, 10), nan_buf(B, 10)

    def forward(self, x, labels, training=True):
        b1, b2, b3, b4, b5, b6, b7 = self.bn
        self.c1.forward(x, self.y1)
        b1.forward(self.y1, self.z1, training=training)
        self.pool.forward(self.z1, self.x2)
        self.c2.forward(self.x2, self.y2)
        b2.forward(self.y2, self.x0, training=training)
        self.c3.forward(self.x0, self.y3)
        b3.forward(self.y3, self.z3, training=training)
        self.c4.forward(self.z3, self.y4)
        b4.forward(self.y4, self.z4, training=training)
        self.se1.forward(self.z4, self.x1, r=self.x0)
        self.c5.forward(self.x1, self.y5)
        b5.forward(self.y5, self.z5, training=training)
        self.c6.forward(self.z5, self.y6)
        self.c7.forward(self.x1, self.y7)
        b7.forward(self.y7, self.s, training=training)
        b6.forward(self.y6, self.z6, training=training)
        self.se2.forward(self.z6, self.out, r=self.s)
        self.gap.forward(self.out, self.h)
        self.fc.forward(self.h, self.z)
        self.eng.softmax_ce_bf16(self.z, labels, self.NB, 10, 1.0 / self.NB, self.dz, self.loss, self.pred)

    def backward(self):
        b1, b2, b3, b4, b5, b6, b7 = self.bn
        self.fc.backward(self.z, self.dz, self.dh)
        self.gap.backward(self.dh, self.dout)
        self.se2.backward(self.out, self.dout, self.dz6, dr=self.ds)
        b6.backward(self.z6, self.dz6, self.dy6)
        self.c6.backward(self.y6, self.dy6, self.dz5)
        b5.backward(self.z5, self.dz5, self.dy5)
        self.c5.backward(self.y5, self.dy5, self.dx1)
        b7.backward(self.s, self.ds, self.dy7)
        self.c7.backward(self.y7, self.dy7, self.dx1p)
        self.se1.backward(self.x1, self.dx1, self.dz4, dr=self.dres, dy2=self.dx1p)   # main path and projection meet at x1
        b4.backward(self.z4, self.dz4, self.dy4)
        self.c4.backward(self.y4, self.dy4, self.dz3)
        b3.backward(self.z3, self.dz3, self.dy3)
        self.c3.backward(self.y3, self.dy3, self.dx0)
        b2.backward(self.x0, self.dx0, self.dy2, dy2=self.dres)
        self.c2.backward(self.y2, self.dy2, self.dx2)
        self.pool.backward(self.dx2, self.dz1)
        b1.backward(self.z1, self.dz1, self.dy1)
        self.c1.backward(self.y1, self.dy1, None)

    def layers(self):
        return (*super().layers(), self.se1, self.se2)


class MobileNetLite(Network):
    """stem conv 48@5x5 -> BN+ReLU (x0) -> [1x1 48->96, BN+ReLU, depthwise 3x3/1 pad 1, BN+ReLU, 1x1 96->48, BN + x0] (x1) ->
    [1x1 48->96, BN+ReLU, depthwise 3x3/2 pad 1, BN+ReLU, 1x1 96->64, BN] -> GAP -> fc 64->10 -> softmax CE (1/B).  The convs have
    no bias; the blocks end without a ReLU (MobileNetV2's linear bottleneck).  Every 1x1 conv reads >= 48 channels, so each is a
    wide-family layer, which has a 1x1 input gradient."""
    LR_STEP, EPOCHS = 0.2, 40
    SEED, PARAMS = 21, [("f0", (48, 5, 5, 1), 25), ("e1", (96, 1, 1, 48), 48), ("d1", (96, 3, 3), 9), ("p1", (48, 1, 1, 96), 96),
                        ("e2", (96, 1, 1, 48), 48), ("d2", (96, 3, 3), 9), ("p2", (64, 1, 1, 96), 96), ("w8", (10, 1, 1, 64), 64),
                        ("b8", 10, 64)]

    def __init__(self, eng, pkg, p):
        super().__init__(eng)
        relu, none = pkg.ACT_RELU, pkg.ACT_NONE
        B = self.NB
        conv = lambda H, C, K, R, f: pkg.ConvLayer(eng, B, H, H, C, K, R, R, p[f], None, act=none)
        self.stem = conv(28, 1, 48, 5, "f0")
        self.e1, self.p1 = conv(24, 48, 96, 1, "e1"), conv(24, 96, 48, 1, "p1")
        self.e2, self.p2 = conv(24, 48, 96, 1, "e2"), conv(12, 96, 64, 1, "p2")
        assert self.stem.family == "narrow" and all(c.family == "wide" for c in (self.e1, self.p1, self.e2, self.p2))
        self.d1 = pkg.DepthwiseConvLayer(eng, B, 24, 24, 96, 3, 3, p["d1"], None, act=none, stride=1, padding=(1, 1))
        self.d2 = pkg.DepthwiseConvLayer(eng, B, 24, 24, 96, 3, 3, p["d2"], None, act=none, stride=2, padding=(1, 1))
        assert self.d1.out_shape == (B, 24, 24, 96) and self.d2.out_shape == (B, 12, 12, 96)
        BN = lambda H, C, act: pkg.BatchNormLayer(eng, B, H, H, C, act=act)
        self.bn = [BN(24, 48, relu), BN(24, 96, relu), BN(24, 96, relu), BN(24, 48, none), BN(24, 96, relu), BN(12, 96, relu),
                   BN(12, 64, none)]
        self.gap = pkg.GlobalAvgPoolLayer(eng, B, 12, 12, 64)
        self.fc = pkg.LinearLayer(eng, B, 1, 1, 64, 10, p["w8"], p["b8"], act=none, row_pitch=self.gap.row_pitch)
        self.y0, self.x0, self.dx0, self.dy0, self.dres, self.yp1, self.x1, self.dx1, self.dyp1 = (nan_buf(B, 24, 24, 48) for _ in range(9))
        (self.ye1, self.ze1, self.yd1, self.zd1, self.dzd1, self.dyd1, self.dze1, self.dye1,
         self.ye2, self.ze2, self.dze2, self.dye2) = (nan_buf(B, 24, 24, 96) for _ in range(12))
        self.yd2, self.zd2, self.dzd2, self.dyd2 = (nan_buf(B, 12, 12, 96) for _ in range(4))
        self.yp2, self.out, self.dout, self.dyp2 = (nan_buf(B, 12, 12, 64) for _ in range(4))
        self.h, self.dh = nan_buf(B, self.gap.row_pitch), nan_buf(B, self.gap.row_pitch)
        self.z, self.dz = nan_buf(B, 10), nan_buf(B, 10)

    def forward(self, x, labels, training=True):
        b0, be1, bd1, bp1, be2, bd2, bp2 = self.bn
        self.stem.forward(x, self.y0)
        b0.forward(self.y0, self.x0, training=training)
        self.e1.forward(self.x0, self.ye1)
        be1.forward(self.ye1, self.ze1, training=training)
        self.d1.forward(self.ze1, self.yd1)
        bd1.forward(self.yd1, self.zd1, training=training)
        self.p1.forward(self.zd1, self.yp1)
        bp1.forward(self.yp1, self.x1, r=self.x0, training=training)
        self.e2.forward(self.x1, self.ye2)
        be2.forward(self.ye2, self.ze2, training=training)
        self.d2.forward(self.ze2, self.yd2)
        bd2.forward(self.yd2, self.zd2, training=training)
        self.p2.forward(self.zd2, self.yp2)
        bp2.forward(self.yp2, self.out, training=training)
        self.gap.forward(self.out, self.h)
        self.fc.forward(self.h, self.z)
        self.eng.softmax_ce_bf16(self.z, labels, self.NB, 10, 1.0 / self.NB, self.dz, self.loss, self.pred)

    def backward(self):
        b0, be1, bd1, bp1, be2, bd2, bp2 = self.bn
        self.fc.backward(self.z, self.dz, self.dh)
        self.gap.backward(self.dh, self.dout)
        bp2.backward(self.out, self.dout, self.dyp2)
        self.p2.backward(self.yp2, self.dyp2, self.dzd2)
        bd2.backward(self.zd2, self.dzd2, self.dyd2)
        self.d2.backward(self.yd2, self.dyd2, self.dze2)
        be2.backward(self.ze2, self.dze2, self.dye2)
        self.e2.backward(self.ye2, self.dye2, self.dx1)
        bp1.backward(self.x1, self.dx1, self.dyp1, dr=self.dres)
        self.p1.backward(self.yp1, self.dyp1, self.dzd1)
        bd1.backward(self.zd1, self.dzd1, self.dyd1)
        self.d1.backward(self.yd1, self.dyd1, self.dze1)
        be1.backward(self.ze1, self.dze1, self.dye1)
        self.e1.backward(self.ye1, self.dye1, self.dx0)
        b0.backward(self.x0, self.dx0, self.dy0, dy2=self.dres)                    # the block's two paths meet at x0
        self.stem.backward(self.y0, self.dy0, None)

    def layers(self):
        return (self.stem, self.e1, self.d1, self.p1, self.e2, self.d2, self.p2, self.fc, *self.bn)

    def stateless(self):
        return (self.gap,)


class EfficientNetLite(Network):
    """stem conv 48@5x5 -> BN+SiLU -> avg pool 2 (12x12x48) -> MBConv [1x1 48->96, BN+ReLU6, depthwise 3x3/2 pad 1, BN+ReLU6,
    1x1 96->48, BN] (x1, 6x6x48) -> MBConv [1x1 48->96, BN+SiLU, depthwise 5x5 pad 2, BN+SiLU, SE 96->8->96, 1x1 96->48, BN + x1]
    -> 1x1 48->128, BN+hard-swish -> GAP -> fc 128->10 -> softmax CE (1/B).  The convs have no bias.  Every 1x1 conv reads >= 48
    channels, so each is a wide-family layer, which has a 1x1 input gradient.  Each new-code BN also writes dr (= g) so that the
    test can read the gradient it formed."""
    LR_STEP, EPOCHS = 0.2, 30
    SEED, PARAMS = 31, [("f0", (48, 5, 5, 1), 25), ("e1", (96, 1, 1, 48), 48), ("d1", (96, 3, 3), 9), ("p1", (48, 1, 1, 96), 96),
                        ("e2", (96, 1, 1, 48), 48), ("d2", (96, 5, 5), 25), ("p2", (48, 1, 1, 96), 96), ("h", (128, 1, 1, 48), 48),
                        ("w8", (10, 1, 1, 128), 128), ("b8", 10, 128),
                        ("s1", (8, 96), 96), ("sb1", 8, 96), ("s2", (96, 8), 8), ("sb2", 96, 8)]

    def __init__(self, eng, pkg, p):
        super().__init__(eng)
        none, silu, hs, r6 = pkg.ACT_NONE, pkg.ACT_SILU, pkg.ACT_HARDSWISH, pkg.ACT_RELU6
        B = self.NB
        conv = lambda H, C, K, R, f: pkg.ConvLayer(eng, B, H, H, C, K, R, R, p[f], None, act=none)
        self.stem = conv(28, 1, 48, 5, "f0")
        self.e1, self.p1 = conv(12, 48, 96, 1, "e1"), conv(6, 96, 48, 1, "p1")
        self.e2, self.p2, self.hd = conv(6, 48, 96, 1, "e2"), conv(6, 96, 48, 1, "p2"), conv(6, 48, 128, 1, "h")
        assert all(c.family == "wide" for c in (self.e1, self.p1, self.e2, self.p2, self.hd))
        self.d1 = pkg.DepthwiseConvLayer(eng, B, 12, 12, 96, 3, 3, p["d1"], None, act=none, stride=2, padding=(1, 1))
        self.d2 = pkg.DepthwiseConvLayer(eng, B, 6, 6, 96, 5, 5, p["d2"], None, act=none, stride=1, padding=(2, 2))
        assert self.d1.out_shape == (B, 6, 6, 96) and self.d2.out_shape == (B, 6, 6, 96)
        self.se = pkg.SqueezeExcitationLayer(eng, B, 6, 6, 96, 8, p["s1"], p["sb1"], p["s2"], p["sb2"], act=none)
        BN = lambda H, C, act: pkg.BatchNormLayer(eng, B, H, H, C, act=act)
        self.bn = [BN(24, 48, silu), BN(12, 96, r6), BN(6, 96, r6), BN(6, 48, none), BN(6, 96, silu), BN(6, 96, silu), BN(6, 48, none),
                   BN(6, 128, hs)]
        self.pool = pkg.AvgPoolLayer(eng, B, 24, 24, 48, 2, row_pitch=self.e1.row_pitch, image_rows=self.e1.image_rows)
        self.gap = pkg.GlobalAvgPoolLayer(eng, B, 6, 6, 128)
        self.fc = pkg.LinearLayer(eng, B, 1, 1, 128, 10, p["w8"], p["b8"], act=none, row_pitch=self.gap.row_pitch)
        self.y0, self.z0, self.dz0, self.dy0, self.g0 = (nan_buf(B, 24, 24, 48) for _ in range(5))
        self.x1p, self.dx1p = nan_buf(B, 12, self.e1.row_pitch), nan_buf(B, 12, self.e1.row_pitch)
        self.ye1, self.ze1, self.dze1, self.dye1, self.ge1 = (nan_buf(B, 12, 12, 96) for _ in range(5))
        (self.yd1, self.zd1, self.dzd1, self.dyd1, self.gd1, self.ye2, self.ze2, self.dze2, self.dye2, self.ge2, self.yd2, self.zd2,
         self.dzd2, self.dyd2, self.gd2, self.se_y, self.dse_y) = (nan_buf(B, 6, 6, 96) for _ in range(17))
        (self.yp1, self.x1, self.dx1, self.dyp1, self.yp2, self.x2, self.dx2, self.dyp2, self.dres, self.dx1b) = (nan_buf(B, 6, 6, 48) for _ in range(10))
        self.yh, self.zh, self.dzh, self.dyh, self.gh = (nan_buf(B, 6, 6, 128) for _ in range(5))
        self.hp, self.dhp = nan_buf(B, self.gap.row_pitch), nan_buf(B, self.gap.row_pitch)
        self.z, self.dz = nan_buf(B, 10), nan_buf(B, 10)

    def forward(self, x, labels, training=True):
        b0, be1, bd1, bp1, be2, bd2, bp2, bh = self.bn
        self.stem.forward(x, self.y0)
        b0.forward(self.y0, self.z0, training=training)
        self.pool.forward(self.z0, self.x1p)
        self.e1.forward(self.x1p, self.ye1)
        be1.forward(self.ye1, self.ze1, training=training)
        self.d1.forward(self.ze1, self.yd1)
        bd1.forward(self.yd1, self.zd1, training=training)
        self.p1.forward(self.zd1, self.yp1)
        bp1.forward(self.yp1, self.x1, training=training)
        self.e2.forward(self.x1, self.ye2)
        be2.forward(self.ye2, self.ze2, training=training)
        self.d2.forward(self.ze2, self.yd2)
        bd2.forward(self.yd2, self.zd2, training=training)
        self.se.forward(self.zd2, self.se_y)
        self.p2.forward(self.se_y, self.yp2)
        bp2.forward(self.yp2, self.x2, r=self.x1, training=training)
        self.hd.forward(self.x2, self.yh)
        bh.forward(self.yh, self.zh, training=training)
        self.gap.forward(self.zh, self.hp)
        self.fc.forward(self.hp, self.z)
        self.eng.softmax_ce_bf16(self.z, labels, self.NB, 10, 1.0 / self.NB, self.dz, self.loss, self.pred)

    def backward(self):
        b0, be1, bd1, bp1, be2, bd2, bp2, bh = self.bn
        self.fc.backward(self.z, self.dz, self.dhp)
        self.gap.backward(self.dhp, self.dzh)
        bh.backward(self.zh, self.dzh, self.dyh, dr=self.gh)
        self.hd.backward(self.yh, self.dyh, self.dx2)
        bp2.backward(self.x2, self.dx2, self.dyp2, dr=self.dres)
        self.p2.backward(self.yp2, self.dyp2, self.dse_y)
        self.se.backward(self.se_y, self.dse_y, self.dzd2)
        bd2.backward(self.zd2, self.dzd2, self.dyd2, dr=self.gd2)
        self.d2.backward(self.yd2, self.dyd2, self.dze2)
        be2.backward(self.ze2, self.dze2, self.dye2, dr=self.ge2)
        self.e2.backward(self.ye2, self.dye2, self.dx1b)
        bp1.backward(self.x1, self.dx1b, self.dyp1, dy2=self.dres)                  # the block's two paths meet at x1
        self.p1.backward(self.yp1, self.dyp1, self.dzd1)
        bd1.backward(self.zd1, self.dzd1, self.dyd1, dr=self.gd1)
        self.d1.backward(self.yd1, self.dyd1, self.dze1)
        be1.backward(self.ze1, self.dze1, self.dye1, dr=self.ge1)
        self.e1.backward(self.ye1, self.dye1, self.dx1p)
        self.pool.backward(self.dx1p, self.dz0)
        b0.backward(self.z0, self.dz0, self.dy0, dr=self.g0)
        self.stem.backward(self.y0, self.dy0, None)

    # (new-code BN layer, its x, y, dy, dx, g) for the replays
    def bn_tensors(self):
        b0, be1, bd1, bp1, be2, bd2, bp2, bh = self.bn
        return [(b0, self.y0, self.z0, self.dz0, self.dy0, self.g0), (be1, self.ye1, self.ze1, self.dze1, self.dye1, self.ge1),
                (bd1, self.yd1, self.zd1, self.dzd1, self.dyd1, self.gd1), (be2, self.ye2, self.ze2, self.dze2, self.dye2, self.ge2),
                (bd2, self.yd2, self.zd2, self.dzd2, self.dyd2, self.gd2), (bh, self.yh, self.zh, self.dzh, self.dyh, self.gh)]

    def layers(self):
        return (self.stem, self.e1, self.d1, self.p1, self.e2, self.d2, self.p2, self.hd, self.fc, self.se, *self.bn)

    def stateless(self):
        return (self.pool, self.gap)


class EfficientNetDropout(EfficientNetLite):
    """EfficientNetLite with both regularisers: element dropout (p = 0.2) in place on the global average pool's output before the
    fc, and stochastic depth (p = 0.2, per image) on the residual MBConv, whose last BN runs without r while the DropoutLayer adds
    x1.  With `trace` the layers' inputs that the in-place calls overwrite are kept."""
    P_FC, P_PATH = 0.2, 0.2
    SEED_FC, SEED_PATH = 1001, 2002

    def __init__(self, eng, pkg, p):
        super().__init__(eng, pkg, p)
        NB = self.NB
        self.drop_fc = pkg.DropoutLayer(eng, NB, 128, self.P_FC, self.SEED_FC, row_pitch=self.gap.row_pitch)
        self.drop_path = pkg.DropoutLayer(eng, NB, 6 * 6 * 48, self.P_PATH, self.SEED_PATH, per_sample=True)
        self.b2, self.db2 = (nan_buf(NB, 6, 6, 48) for _ in range(2))
        self.trace = False

    def snapshot(self, t):
        """a copy of t as the engine's stream has written it, taken before the engine's next call overwrites it (torch copies on
        its own stream)"""
        self.eng.sync()
        copy = t.clone()
        torch.cuda.synchronize()
        return copy

    def forward(self, x, labels, training=True):
        b0, be1, bd1, bp1, be2, bd2, bp2, bh = self.bn
        self.stem.forward(x, self.y0)
        b0.forward(self.y0, self.z0, training=training)
        self.pool.forward(self.z0, self.x1p)
        self.e1.forward(self.x1p, self.ye1)
        be1.forward(self.ye1, self.ze1, training=training)
        self.d1.forward(self.ze1, self.yd1)
        bd1.forward(self.yd1, self.zd1, training=training)
        self.p1.forward(self.zd1, self.yp1)
        bp1.forward(self.yp1, self.x1, training=training)
        self.e2.forward(self.x1, self.ye2)
        be2.forward(self.ye2, self.ze2, training=training)
        self.d2.forward(self.ze2, self.yd2)
        bd2.forward(self.yd2, self.zd2, training=training)
        self.se.forward(self.zd2, self.se_y)
        self.p2.forward(self.se_y, self.yp2)
        bp2.forward(self.yp2, self.b2, training=training)                          # the branch's last BN, without r
        self.drop_path.forward(self.b2, self.x2, r=self.x1, training=training)       # x2 = x1 + drop_path(b2)
        self.hd.forward(self.x2, self.yh)
        bh.forward(self.yh, self.zh, training=training)
        self.gap.forward(self.zh, self.hp)
        if self.trace:
            self.hp_in = self.snapshot(self.hp)
        self.drop_fc.forward(self.hp, self.hp, training=training)
        self.fc.forward(self.hp, self.z)
        self.eng.softmax_ce_bf16(self.z, labels, self.NB, 10, 1.0 / self.NB, self.dz, self.loss, self.pred)

    def backward(self):
        b0, be1, bd1, bp1, be2, bd2, bp2, bh = self.bn
        self.fc.backward(self.z, self.dz, self.dhp)
        if self.trace:
            self.dhp_in = self.snapshot(self.dhp)
        self.drop_fc.backward(self.dhp, self.dhp)
        self.gap.backward(self.dhp, self.dzh)
        bh.backward(self.zh, self.dzh, self.dyh, dr=self.gh)
        self.hd.backward(self.yh, self.dyh, self.dx2)
        self.drop_path.backward(self.dx2, self.db2)                                  # dx2 still feeds the skip path
        bp2.backward(self.b2, self.db2, self.dyp2)
        self.p2.backward(self.yp2, self.dyp2, self.dse_y)
        self.se.backward(self.se_y, self.dse_y, self.dzd2)
        bd2.backward(self.zd2, self.dzd2, self.dyd2, dr=self.gd2)
        self.d2.backward(self.yd2, self.dyd2, self.dze2)
        be2.backward(self.ze2, self.dze2, self.dye2, dr=self.ge2)
        self.e2.backward(self.ye2, self.dye2, self.dx1b)
        bp1.backward(self.x1, self.dx1b, self.dyp1, dy2=self.dx2)                   # the block's two paths meet at x1
        self.p1.backward(self.yp1, self.dyp1, self.dzd1)
        bd1.backward(self.zd1, self.dzd1, self.dyd1, dr=self.gd1)
        self.d1.backward(self.yd1, self.dyd1, self.dze1)
        be1.backward(self.ze1, self.dze1, self.dye1, dr=self.ge1)
        self.e1.backward(self.ye1, self.dye1, self.dx1p)
        self.pool.backward(self.dx1p, self.dz0)
        b0.backward(self.z0, self.dz0, self.dy0, dr=self.g0)
        self.stem.backward(self.y0, self.dy0, None)

    def stateless(self):
        return (*super().stateless(), self.drop_fc, self.drop_path)


class ResNeXtLite(Network):
    """stem conv 48@5x5 -> BN+ReLU (x0) -> [1x1 48->64, BN+ReLU, grouped 3x3/1 pad 1 G = 8 (Cg = 8), BN+ReLU, 1x1 64->48,
    BN + x0 with ReLU] (x1) -> [1x1 48->96, BN+ReLU, grouped 3x3/2 pad 1 G = 24 (Cg = 4, the narrow path), BN+ReLU, 1x1 96->64, BN]
    -> GAP -> fc 64->10 -> softmax CE (1/B).  The convs have no bias.  Every 1x1 conv reads >= 48 channels, so each is a
    wide-family layer, which has a 1x1 input gradient."""
    LR_STEP, EPOCHS = 0.2, 40
    SEED, PARAMS = 23, [("f0", (48, 5, 5, 1), 25), ("e1", (64, 1, 1, 48), 48), ("g1", (64, 3, 3, 8), 72), ("p1", (48, 1, 1, 64), 64),
                        ("e2", (96, 1, 1, 48), 48), ("g2", (96, 3, 3, 4), 36), ("p2", (64, 1, 1, 96), 96), ("w8", (10, 1, 1, 64), 64),
                        ("b8", 10, 64)]

    def __init__(self, eng, pkg, p):
        super().__init__(eng)
        relu, none = pkg.ACT_RELU, pkg.ACT_NONE
        B = self.NB
        conv = lambda H, C, K, R, f: pkg.ConvLayer(eng, B, H, H, C, K, R, R, p[f], None, act=none)
        self.stem = conv(28, 1, 48, 5, "f0")
        self.e1, self.p1 = conv(24, 48, 64, 1, "e1"), conv(24, 64, 48, 1, "p1")
        self.e2, self.p2 = conv(24, 48, 96, 1, "e2"), conv(12, 96, 64, 1, "p2")
        assert self.stem.family == "narrow" and all(c.family == "wide" for c in (self.e1, self.p1, self.e2, self.p2))
        self.g1 = pkg.GroupedConvLayer(eng, B, 24, 24, 64, 64, 8, 3, 3, p["g1"], None, act=none, stride=1, padding=(1, 1))
        self.g2 = pkg.GroupedConvLayer(eng, B, 24, 24, 96, 96, 24, 3, 3, p["g2"], None, act=none, stride=2, padding=(1, 1))
        assert self.g1.out_shape == (B, 24, 24, 64) and self.g2.out_shape == (B, 12, 12, 96)
        assert self.g1.info["vec"] == 8 and self.g2.info["vec"] == 4
        BN = lambda H, C, act: pkg.BatchNormLayer(eng, B, H, H, C, act=act)
        self.bn = [BN(24, 48, relu), BN(24, 64, relu), BN(24, 64, relu), BN(24, 48, relu), BN(24, 96, relu), BN(12, 96, relu),
                   BN(12, 64, none)]
        self.gap = pkg.GlobalAvgPoolLayer(eng, B, 12, 12, 64)
        self.fc = pkg.LinearLayer(eng, B, 1, 1, 64, 10, p["w8"], p["b8"], act=none, row_pitch=self.gap.row_pitch)
        self.y0, self.x0, self.dx0, self.dy0, self.dres, self.yp1, self.x1, self.dx1, self.dyp1 = (nan_buf(B, 24, 24, 48) for _ in range(9))
        self.ye1, self.ze1, self.yg1, self.zg1, self.dzg1, self.dyg1, self.dze1, self.dye1 = (nan_buf(B, 24, 24, 64) for _ in range(8))
        self.ye2, self.ze2, self.dze2, self.dye2 = (nan_buf(B, 24, 24, 96) for _ in range(4))
        self.yg2, self.zg2, self.dzg2, self.dyg2 = (nan_buf(B, 12, 12, 96) for _ in range(4))
        self.yp2, self.out, self.dout, self.dyp2 = (nan_buf(B, 12, 12, 64) for _ in range(4))
        self.h, self.dh = nan_buf(B, self.gap.row_pitch), nan_buf(B, self.gap.row_pitch)
        self.z, self.dz = nan_buf(B, 10), nan_buf(B, 10)

    def forward(self, x, labels, training=True):
        b0, be1, bg1, bp1, be2, bg2, bp2 = self.bn
        self.stem.forward(x, self.y0)
        b0.forward(self.y0, self.x0, training=training)
        self.e1.forward(self.x0, self.ye1)
        be1.forward(self.ye1, self.ze1, training=training)
        self.g1.forward(self.ze1, self.yg1)
        bg1.forward(self.yg1, self.zg1, training=training)
        self.p1.forward(self.zg1, self.yp1)
        bp1.forward(self.yp1, self.x1, r=self.x0, training=training)
        self.e2.forward(self.x1, self.ye2)
        be2.forward(self.ye2, self.ze2, training=training)
        self.g2.forward(self.ze2, self.yg2)
        bg2.forward(self.yg2, self.zg2, training=training)
        self.p2.forward(self.zg2, self.yp2)
        bp2.forward(self.yp2, self.out, training=training)
        self.gap.forward(self.out, self.h)
        self.fc.forward(self.h, self.z)
        self.eng.softmax_ce_bf16(self.z, labels, self.NB, 10, 1.0 / self.NB, self.dz, self.loss, self.pred)

    def backward(self):
        b0, be1, bg1, bp1, be2, bg2, bp2 = self.bn
        self.fc.backward(self.z, self.dz, self.dh)
        self.gap.backward(self.dh, self.dout)
        bp2.backward(self.out, self.dout, self.dyp2)
        self.p2.backward(self.yp2, self.dyp2, self.dzg2)
        bg2.backward(self.zg2, self.dzg2, self.dyg2)
        self.g2.backward(self.yg2, self.dyg2, self.dze2)
        be2.backward(self.ze2, self.dze2, self.dye2)
        self.e2.backward(self.ye2, self.dye2, self.dx1)
        bp1.backward(self.x1, self.dx1, self.dyp1, dr=self.dres)
        self.p1.backward(self.yp1, self.dyp1, self.dzg1)
        bg1.backward(self.zg1, self.dzg1, self.dyg1)
        self.g1.backward(self.yg1, self.dyg1, self.dze1)
        be1.backward(self.ze1, self.dze1, self.dye1)
        self.e1.backward(self.ye1, self.dye1, self.dx0)
        b0.backward(self.x0, self.dx0, self.dy0, dy2=self.dres)                    # the block's two paths meet at x0
        self.stem.backward(self.y0, self.dy0, None)

    def layers(self):
        return (self.stem, self.e1, self.g1, self.p1, self.e2, self.g2, self.p2, self.fc, *self.bn)

    def stateless(self):
        return (self.gap,)


def train(eng, pkg, golden, make, epochs, update=None, batches=None, tests=None, check_step=None, check_trained=None):
    """The end-to-end schedule of make()'s network (B = its NB), returning (mean loss of each epoch, test accuracy, the parameters
    after 5 steps):
    1. a fresh network takes the first 5 steps of `batches`' epoch 0: check_step(net, it, x, labels) runs the forward and backward
       of each (default: without checks), then update(net) (default: net.sgd(net.LR_STEP)) and eng.sync();
    2. a second fresh network trains for `epochs` epochs; after its step 5 its parameters equal the first's bit for bit;
    3. check_trained(net) after the last step; eval with training=False over `tests`; check_trained(net) again.
    `batches` and `tests` default to Slices of the golden training and test digits; an ImageBatcher fits in either.  Each network is
    closed, also when a check fails.  The engine runs on its own stream; the fresh loss buffer of each step and the networks' NaN
    fills run on torch's."""
    update = update or (lambda net: net.sgd(net.LR_STEP))
    if check_step is None:
        def check_step(net, it, x, labels):
            net.forward(x, labels)
            net.backward()
    net = make()
    try:
        B = net.NB
        batches = batches or Slices(pkg, golden["train_u8"], golden["train_labels"], B)
        tests = tests or Slices(pkg, golden["test_u8"], golden["test_labels"], B)
        batches.epoch = 0
        for it in range(5):
            check_step(net, it, *batches.batch(it))
            update(net)
            eng.sync()
        after5 = net.params()
    finally:
        net.close()

    net = make()
    try:
        losses, spe = [], batches.steps_per_epoch
        for ep in range(epochs):
            batches.epoch = ep
            for s in range(spe):
                net.forward(*batches.batch(s))
                net.backward()
                update(net)
                losses.append(net.loss)
                net.loss = torch.zeros(B, dtype=torch.float32, device=DEV)
                if ep == 0 and s == 4:
                    eng.sync()
                    assert same_bits(net.params(), after5)
        eng.sync()
        ep_loss = [float(torch.stack(losses[e * spe:(e + 1) * spe]).double().mean()) for e in range(epochs)]
        if check_trained:
            check_trained(net)
        right = 0
        for s in range(tests.steps_per_epoch):
            net.forward(*tests.batch(s, training=False), training=False)
            eng.sync()
            right += int((net.pred.cpu().numpy() == golden["test_labels"][s * B:(s + 1) * B]).sum())
        if check_trained:
            check_trained(net)
    finally:
        net.close()
    return ep_loss, right / (tests.steps_per_epoch * B), after5
