"""A DeepLab-style segmenter trained on the golden digits (TEST INFRASTRUCTURE ONLY) with segment_nets' harness
(segment_nets.train_segmenter): after the stem the map keeps its 14 x 14 resolution, and dilated ("atrous") convolutions widen the
receptive field in place of further striding.  The targets are segment_ref.digit_masks: 11 classes, 255 ignored."""
import torch

from example_nets import DEV, Network, nan_buf
import segment_nets
from segment_nets import O, _Segmenter

# name, shape, fan_in: KRSC filters of the wide / row-Toeplitz layers, [C][R][S] for the depthwise one
DEEPLAB_PARAMS = segment_nets.ENCODER[:2] + [
    ("fd1", (32, 3, 3, 32), 288), ("fd2", (32, 3, 3, 32), 288),      # the dilated block
    ("fa", (32, 1, 1, 32), 32), ("fb", (32, 3, 3, 32), 288),         # ASPP: 1x1 (a per-pixel fc), 3x3 at dilation 4
    ("wc", (32, 3, 3), 9), ("fp", (32, 1, 1, 32), 32),               # ASPP: 3x3 depthwise at dilation 6, then 1x1
    ("w", (O, 1, 1, 32), 32), ("bw", O, 32)]


class DeepLabLite(_Segmenter):
    """stem: conv 16@3x3 pad 1 -> BN+ReLU (a, 28x28) -> conv 32@3x3/2 pad 1 -> BN+ReLU (b, 14x14)
    dilated block: conv 32@3x3 dil 2 pad 2 -> BN+ReLU (m) -> conv 32@3x3 dil 2 pad 2 -> BN + b -> ReLU (h)
    ASPP-lite head, three branches each followed by a batch norm and summed through its residual input:
        sa = BN(conv 1x1 (m)),  sb = BN(conv 3x3 dil 4 pad 4 (h)) + sa,  out = ReLU(BN(conv 1x1 (depthwise 3x3 dil 6 pad 6 (h))) + sb)
    output: per-pixel fc 32->11 at 14x14 -> bilinear 14x14 -> 28x28 -> per-pixel CE (ignore 255).  No conv has a bias.
    The 1x1 convolutions are per-pixel fully connected layers (LinearLayer over the N*14*14 pixels), as the output head is.
    The 1x1 branch reads the block's middle activation m rather than h, so that every activation feeds at most two layers and batch
    norm's second incoming gradient (dy2) joins their gradients: h's two readers join at the block's last batch norm, m's at its
    first."""
    SEED = 41
    PARAMS = DEEPLAB_PARAMS

    def __init__(self, eng, pkg, p):
        Network.__init__(self, eng)                      # _Segmenter.__init__ would build FCN's third encoder stage
        B, relu = self.NB, pkg.ACT_RELU
        self.pixels = B * 28 * 28
        self.loss = torch.zeros(self.pixels, dtype=torch.float32, device=DEV)
        self.pred = torch.zeros(self.pixels, dtype=torch.int32, device=DEV)
        self.count = torch.zeros(1, dtype=torch.int32, device=DEV)
        self.c1 = pkg.ConvLayer(eng, B, 28, 28, 8, 16, 3, 3, p["f1"], padding=(1, 1))
        self.c2 = pkg.ConvLayer(eng, B, 28, 28, 16, 32, 3, 3, p["f2"], padding=(1, 1), stride=2)
        self.bn1 = pkg.BatchNormLayer(eng, B, 28, 28, 16, act=relu)
        self.bn2 = pkg.BatchNormLayer(eng, B, 14, 14, 32, act=relu)
        self.d1 = pkg.ConvLayer(eng, B, 14, 14, 32, 32, 3, 3, p["fd1"], padding=(2, 2), dilation=(2, 2))
        self.d2 = pkg.ConvLayer(eng, B, 14, 14, 32, 32, 3, 3, p["fd2"], padding=(2, 2), dilation=(2, 2))
        self.ca = pkg.LinearLayer(eng, B * 196, 1, 1, 32, 32, p["fa"], row_pitch=32)
        self.cb = pkg.ConvLayer(eng, B, 14, 14, 32, 32, 3, 3, p["fb"], padding=(4, 4), dilation=(4, 4))
        self.cc = pkg.DepthwiseConvLayer(eng, B, 14, 14, 32, 3, 3, p["wc"], padding=(6, 6), dilation=(6, 6))
        self.cp = pkg.LinearLayer(eng, B * 196, 1, 1, 32, 32, p["fp"], row_pitch=32)
        self.bnd1 = pkg.BatchNormLayer(eng, B, 14, 14, 32, act=relu)
        self.bnd2 = pkg.BatchNormLayer(eng, B, 14, 14, 32, act=relu)
        self.bna = pkg.BatchNormLayer(eng, B, 14, 14, 32)
        self.bnb = pkg.BatchNormLayer(eng, B, 14, 14, 32)
        self.bnc = pkg.BatchNormLayer(eng, B, 14, 14, 32, act=relu)
        self.fc = pkg.LinearLayer(eng, B * 196, 1, 1, 32, O, p["w"], p["bw"], row_pitch=32)
        self.up = pkg.UpsampleBilinearLayer(eng, B, 14, 14, O, 28, 28)
        self.y1, self.a, self.dy1, self.da = (nan_buf(B, 28, 28, 16) for _ in range(4))
        (self.y2, self.b, self.dy2, self.db, self.db_res, self.yd1, self.m, self.dyd1, self.dm, self.dm_a, self.yd2, self.h, self.dyd2,
         self.dh_b, self.dh_c, self.ya, self.sa, self.dya, self.dsa, self.yb, self.sb, self.dyb, self.dsb, self.yc, self.dyc, self.yp,
         self.out, self.dyp, self.dout) = (nan_buf(B, 14, 14, 32) for _ in range(29))
        self.z14, self.dz14 = nan_buf(B * 196, O), nan_buf(B * 196, O)
        self.z, self.dz = nan_buf(self.pixels, O), nan_buf(self.pixels, O)

    def forward(self, x, labels, masks, training=True):
        self.c1.forward(x, self.y1)
        self.bn1.forward(self.y1, self.a, training=training)
        self.c2.forward(self.a, self.y2)
        self.bn2.forward(self.y2, self.b, training=training)
        self.d1.forward(self.b, self.yd1)
        self.bnd1.forward(self.yd1, self.m, training=training)
        self.d2.forward(self.m, self.yd2)
        self.bnd2.forward(self.yd2, self.h, r=self.b, training=training)
        self.ca.forward(self.m, self.ya)
        self.bna.forward(self.ya, self.sa, training=training)
        self.cb.forward(self.h, self.yb)
        self.bnb.forward(self.yb, self.sb, r=self.sa, training=training)
        self.cc.forward(self.h, self.yc)
        self.cp.forward(self.yc, self.yp)
        self.bnc.forward(self.yp, self.out, r=self.sb, training=training)
        self.fc.forward(self.out, self.z14)
        self.up.forward(self.z14, self.z)
        self.pixel_loss(self.z, masks)

    def backward(self):
        self.up.backward(self.dz, self.dz14)
        self.fc.backward(self.z14, self.dz14, self.dout)
        self.bnc.backward(self.out, self.dout, self.dyp, dr=self.dsb)
        self.cp.backward(self.yp, self.dyp, self.dyc)
        self.cc.backward(self.yc, self.dyc, self.dh_c)
        self.bnb.backward(self.sb, self.dsb, self.dyb, dr=self.dsa)
        self.cb.backward(self.yb, self.dyb, self.dh_b)
        self.bna.backward(self.sa, self.dsa, self.dya)
        self.ca.backward(self.ya, self.dya, self.dm_a)
        self.bnd2.backward(self.h, self.dh_b, self.dyd2, dr=self.db_res, dy2=self.dh_c)
        self.d2.backward(self.yd2, self.dyd2, self.dm)
        self.bnd1.backward(self.m, self.dm, self.dyd1, dy2=self.dm_a)
        self.d1.backward(self.yd1, self.dyd1, self.db)
        self.bn2.backward(self.b, self.db, self.dy2, dy2=self.db_res)
        self.c2.backward(self.y2, self.dy2, self.da)
        self.bn1.backward(self.a, self.da, self.dy1)
        self.c1.backward(self.y1, self.dy1, None)

    def dilated(self):
        """the dilated layers: (layer, its input, its output, the gradient its last backward consumed, its dx)"""
        return ((self.d1, self.b, self.yd1, self.dyd1, self.db), (self.d2, self.m, self.yd2, self.dyd2, self.dm),
                (self.cb, self.h, self.yb, self.dyb, self.dh_b), (self.cc, self.h, self.yc, self.dyc, self.dh_c))

    def layers(self):
        return (self.c1, self.c2, self.bn1, self.bn2, self.d1, self.d2, self.bnd1, self.bnd2, self.ca, self.cb, self.cc, self.cp, self.bna,
                self.bnb, self.bnc, self.fc)

    def stateless(self):
        return (self.up,)
