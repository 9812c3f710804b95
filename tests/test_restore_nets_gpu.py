"""The two restorers of restore_nets.py trained end to end on the H100: in each of the first five steps the pixel shuffle, the pixel
unshuffle and the regression loss are checked bit for bit on the device's own operands; a fresh run reproduces the parameters after
five steps; the test PSNR comes within 1 dB of the float32 CPU replica's and beats the network's baseline."""
import numpy as np
import pytest

import restore_nets
import restore_ref as RR
from example_nets import host

pytestmark = pytest.mark.gpu

# test PSNR (dB) of the float32 torch CPU replicas on the same batches and masks (scripts/restore_replica.py), with the baselines'
REPLICA_PSNR = {"ESPCNLite": 24.39, "DenoiseNet": 23.85}


@pytest.mark.parametrize("name", ["ESPCNLite", "DenoiseNet"])
def test_restorer_trains(pkg, eng, golden, name):
    cls = getattr(restore_nets, name)
    B = cls.NB

    def check_step(net, it, x, xarr):
        net.forward(x)
        eng.sync()
        xb = xarr.to_host().reshape(-1, restore_nets.C_IN)
        assert np.array_equal(host(net.out).reshape(B, 28, 28, 1), RR.shuffle(host(net.z).reshape(B, 14, 14, 4), 2))
        mode = RR.MSE if name == "ESPCNLite" else RR.L1
        g, lw = RR.loss_replay(host(net.out), xb, 1, mode, 1.0 / net.pixels, target_stride=restore_nets.C_IN)
        assert np.array_equal(host(net.dout).reshape(-1), g.reshape(-1))
        assert np.array_equal(net.loss.cpu().numpy().view(np.uint32), lw.view(np.uint32))
        if name == "DenoiseNet":
            assert np.array_equal(host(net.u).reshape(B, 14, 14, 64), RR.unshuffle(host(net.a).reshape(B, 28, 28, 16), 2))
        net.backward()
        eng.sync()
        assert np.any(host(net.dout) != 0)
        assert np.array_equal(host(net.dz).reshape(B, 14, 14, 4), RR.unshuffle(host(net.dout).reshape(B, 28, 28, 1), 2))
        if name == "DenoiseNet":
            assert np.array_equal(host(net.da).reshape(B, 28, 28, 16), RR.shuffle(host(net.du).reshape(B, 14, 14, 64), 2))

    losses, score, base, _ = restore_nets.train_restorer(eng, pkg, golden, cls, check_step)
    print(f"{name}: epoch losses {losses}, test PSNR {score:.2f} dB (replica {REPLICA_PSNR[name]:.2f} dB), baseline {base:.2f} dB")
    assert losses[-1] < losses[0]
    assert score > base
    assert abs(score - REPLICA_PSNR[name]) <= 1.0
