"""ResNetGAP with a non-local block (TEST INFRASTRUCTURE ONLY), trained on the golden digits with example_nets.train: the
self-attention layer inside a real network, with its residual through batch normalization's r and dy2."""
import numpy as np

from example_nets import ResNetGAP, fan_uniform, nan_buf


class NonLocalResNet(ResNetGAP):
    """ResNetGAP (tests/example_nets.py) with a non-local block (Wang et al. 2018) on the 12 x 12 x 16 output x1 of its first
    residual block: T = 144 tokens (two full 64-row key blocks and a ragged 16), one head of d = 16.

        attn.forward(x1, wz);  bn8.forward(wz, x1n, r=x1)        (BN without activation: x1n = BN(W_z y) + x1)

    and the stride-2 stage reads x1n where ResNetGAP's read x1.  In the backward the two stride-2 convolutions' input gradients
    meet in bn8 (dy and dy2); bn8's dr carries them past the block, and the attention's input gradient joins them in the
    BatchNormLayer that wrote x1 (its dy2).  bn8's gamma starts at 0, as in the paper: the block is the identity at step 0 and its
    dO is zero, and from step 1 on gamma, and with it dO, is nonzero.  ResNetGAP's masters, then the block's (w_qkv [48][16], b_qkv,
    w_out [16][16], b_out) from a second generator."""
    NL_SEED, HEADS, HEAD_DIM = 12, 1, 16
    NL_PARAMS = [("nl_wqkv", (48, 16), 16), ("nl_bqkv", 48, 16), ("nl_wout", (16, 16), 16), ("nl_bout", 16, 16)]

    @classmethod
    def init_params(cls):
        return {**super().init_params(), **fan_uniform(cls.NL_SEED, cls.NL_PARAMS)}

    def __init__(self, eng, pkg, p):
        super().__init__(eng, pkg, p)
        B = self.NB
        self.attn = pkg.SelfAttentionLayer(eng, B, 12, 12, 16, self.HEADS, self.HEAD_DIM, p["nl_wqkv"], p["nl_bqkv"], p["nl_wout"],
                                           p["nl_bout"])
        self.bn8 = pkg.BatchNormLayer(eng, B, 12, 12, 16, act=pkg.ACT_NONE, gamma=np.zeros(16, np.float32))
        self.wz, self.x1n, self.dx1n, self.dx1np, self.dwz, self.dnl, self.dxa = (nan_buf(B, 12, 12, 16) for _ in range(7))

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
        self.attn.forward(self.x1, self.wz)
        self.bn8.forward(self.wz, self.x1n, r=self.x1, training=training)
        self.c5.forward(self.x1n, self.y5)
        b5.forward(self.y5, self.z5, training=training)
        self.c6.forward(self.z5, self.y6)
        self.c7.forward(self.x1n, self.y7)
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
        self.c5.backward(self.y5, self.dy5, self.dx1n)
        b7.backward(self.s, self.ds, self.dy7)
        self.c7.backward(self.y7, self.dy7, self.dx1np)
        self.bn8.backward(self.x1n, self.dx1n, self.dwz, dr=self.dnl, dy2=self.dx1np)   # the stride-2 stage meets at x1n
        self.attn.backward(self.dwz, self.dxa)
        b4.backward(self.x1, self.dxa, self.dy4, dr=self.dres, dy2=self.dnl)          # attention and the residual meet at x1
        self.c4.backward(self.y4, self.dy4, self.dz3)
        b3.backward(self.z3, self.dz3, self.dy3)
        self.c3.backward(self.y3, self.dy3, self.dx0)
        b2.backward(self.x0, self.dx0, self.dy2, dy2=self.dres)
        self.c2.backward(self.y2, self.dy2, self.dx2)
        self.pool.backward(self.dx2, self.dz1)
        b1.backward(self.z1, self.dz1, self.dy1)
        self.c1.backward(self.y1, self.dy1, None)

    def layers(self):
        return (*super().layers(), self.attn, self.bn8)
