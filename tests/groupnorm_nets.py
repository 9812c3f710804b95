"""DeepLabLite with group normalization (TEST INFRASTRUCTURE ONLY), trained at a batch of 4 images with segment_nets' harness
(segment_nets.train_segmenter): the regime where batch statistics come from very few samples and group normalization is the usual
choice.  The targets are segment_ref.digit_masks: 11 classes, 255 ignored."""
from deeplab_nets import DeepLabLite


class DeepLabGN(DeepLabLite):
    """DeepLabLite (tests/deeplab_nets.py) with every BatchNormLayer replaced by a GroupNormLayer of GROUPS = 8 groups, at the same
    activation: Cg = 2 channels per group at 16 channels and 4 at 32, so the 16-byte vectors of the kernels span several groups.
    The residual sums of the ASPP-lite head and of the dilated block go through group normalization's r, as they went through
    batch normalization's.  The normalization layers keep DeepLabLite's attribute names (bn1, ..., bnc), so its backward, its
    layer list and its dilated() run unchanged.

    LR and EPOCHS come from the float32 replica (scripts/deeplab_gn_replica.py) at NB = 4, where the harness takes 256 steps per
    epoch: over 8 epochs lr 0.02 reached a test mIoU of 0.519, against 0.483 at 0.01 and 0.493 at 0.05; 16 epochs at 0.02 reach
    0.654."""
    SEED = 43
    NB, LR, EPOCHS = 4, 0.02, 16
    GROUPS = 8
    NORMS = ("bn1", "bn2", "bnd1", "bnd2", "bna", "bnb", "bnc")

    def __init__(self, eng, pkg, p):
        super().__init__(eng, pkg, p)
        for name in self.NORMS:
            bn = getattr(self, name)
            N, H, W, C = bn.shape
            setattr(self, name, pkg.GroupNormLayer(eng, N, H, W, C, self.GROUPS, act=bn.act))
            bn.close()

    def forward(self, x, labels, masks, training=True):
        """DeepLabLite's forward; group normalization computes the same y in training and in evaluation, so `training` reaches no
        layer"""
        self.c1.forward(x, self.y1)
        self.bn1.forward(self.y1, self.a)
        self.c2.forward(self.a, self.y2)
        self.bn2.forward(self.y2, self.b)
        self.d1.forward(self.b, self.yd1)
        self.bnd1.forward(self.yd1, self.m)
        self.d2.forward(self.m, self.yd2)
        self.bnd2.forward(self.yd2, self.h, r=self.b)
        self.ca.forward(self.m, self.ya)
        self.bna.forward(self.ya, self.sa)
        self.cb.forward(self.h, self.yb)
        self.bnb.forward(self.yb, self.sb, r=self.sa)
        self.cc.forward(self.h, self.yc)
        self.cp.forward(self.yc, self.yp)
        self.bnc.forward(self.yp, self.out, r=self.sb)
        self.fc.forward(self.out, self.z14)
        self.up.forward(self.z14, self.z)
        self.pixel_loss(self.z, masks)

    def norms(self):
        """each group normalization with its operands in the last step: (layer, x, r, y, dy, dy2, dx, dr), None where it has none"""
        return ((self.bn1, self.y1, None, self.a, self.da, None, self.dy1, None),
                (self.bn2, self.y2, None, self.b, self.db, self.db_res, self.dy2, None),
                (self.bnd1, self.yd1, None, self.m, self.dm, self.dm_a, self.dyd1, None),
                (self.bnd2, self.yd2, self.b, self.h, self.dh_b, self.dh_c, self.dyd2, self.db_res),
                (self.bna, self.ya, None, self.sa, self.dsa, None, self.dya, None),
                (self.bnb, self.yb, self.sa, self.sb, self.dsb, None, self.dyb, self.dsa),
                (self.bnc, self.yp, self.sb, self.out, self.dout, None, self.dyp, self.dsb))
