"""NonLocalResNet (tests/attention_nets.py) trained on the device with example_nets.train.

- Steps 0-4: each of the first five steps checks the attention core on the device's own operands. The operands are the qkv
  projection's output, o, lse, the dO the output projection wrote, and the dq/dk/dv block it handed back. The checked values are
  o and lse of the forward and dq, dk, dv of the backward, against attention_ref's float64 reference within its bounds.
- Step 0 runs with bn8's gamma at 0, so dO, and with it dq, dk and dv, is exactly zero. Steps 1-4 must see a nonzero dO.
- After five steps, a fresh run must reproduce the parameters bit for bit. train() checks this.
- After training, test accuracy must be within 0.03 of the float32 replica's (scripts/nonlocal_replica.py)."""
import numpy as np
import pytest

import attention_nets
import attention_ref as A
from example_nets import host, train

pytestmark = pytest.mark.gpu

REPLICA_ACC = 0.9297    # scripts/nonlocal_replica.py, lr 0.2, 40 epochs


def check_core(pkg, layer):
    """o, lse, dq, dk and dv of the layer's last step against float64 on its own operands; returns (worst ratios, max |dO|)"""
    N, H, W, C = layer.shape
    h, d, T = layer.heads, layer.d, layer.T
    f = lambda a: pkg.bf16_bits_to_f32(a.to_host().astype(np.uint16)).astype(np.float64)
    qkv, o, do, dqkv = f(layer.qkv_y), f(layer.o), f(layer.do), f(layer.dqkv)
    qkv, dqkv = qkv.reshape(N, T, 3, h, d), dqkv.reshape(N, T, 3, h, d)
    b = A.bounds(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], do.reshape(N, T, h, d), layer.scale)
    got = dict(o=o.reshape(N, T, h, d), lse=layer.lse.to_host().reshape(N, h, T), dq=dqkv[:, :, 0], dk=dqkv[:, :, 1], dv=dqkv[:, :, 2])
    return {name: A.worst(got[name], ref, bound) for name, (ref, bound) in b.items()}, float(np.abs(do).max())


def test_nonlocal_resnet_mnist(eng, pkg, golden):
    cls = attention_nets.NonLocalResNet
    checked, worst, dmax = [], {}, []

    def check_step(net, it, x, labels):
        net.forward(x, labels)
        net.backward()
        eng.sync()
        w, m = check_core(pkg, net.attn)
        for k, v in w.items():
            worst[k] = max(worst.get(k, 0.0), v)
        dmax.append(m)
        assert not np.any((host(net.dxa) & 0x7FFF) > 0x7F80)            # the block's input gradient is finite
        checked.append(it)

    ep_loss, acc, _ = train(eng, pkg, golden, lambda: cls(eng, pkg, cls.init_params()), cls.EPOCHS, check_step=check_step)
    print(f"NonLocalResNet: epoch losses {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}, test accuracy {acc:.4f} (replica {REPLICA_ACC}); "
          f"worst ratios to the bounds {worst}; max |dO| per step {dmax}")
    assert checked == [0, 1, 2, 3, 4]
    assert max(worst.values()) <= 1.0, worst
    assert dmax[0] == 0.0 and all(m > 0 for m in dmax[1:]), dmax
    assert ep_loss[-1] < ep_loss[0]
    assert abs(acc - REPLICA_ACC) <= 0.03
