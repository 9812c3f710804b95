"""ConvVAE of vae_nets.py trained end to end on the H100: in each of the first five steps the Gaussian latent's z, kl and dstats and
the binary cross-entropy's loss and dlogits are checked bit for bit on the device's own operands; a fresh run reproduces the
parameters after five steps; the test negative ELBO comes within a stated tolerance of the float32 CPU replica's, beats the
mean-image baseline by a stated margin, and keeps a KL floor (the latent is used, not collapsed)."""
import numpy as np
import pytest

import vae_nets
import vae_ref as V
from example_nets import host
from restore_nets import C_IN

pytestmark = pytest.mark.gpu

# test negative ELBO per image in nats of the float32 torch CPU replica on the same batches and eps (scripts/vae_replica.py:
# reconstruction 118.13, KL 21.58; the mean-image baseline 198.90)
REPLICA_NELBO = 139.72
# The device and the replica differ by bf16 activations and weights on the device, about 1 % of a loss of this size in the
# other example networks; 3 % of the ELBO leaves room for that and for the fixed single-draw Monte-Carlo estimate.
NELBO_RTOL = 0.03
BASELINE_MARGIN = 40.0        # nats per image below the mean-image baseline
KL_FLOOR = 5.0                # nats per image: a collapsed posterior has KL near 0


def test_conv_vae_trains(pkg, eng, golden):
    cls = vae_nets.ConvVAE
    B, L = cls.NB, cls.L

    def check_step(net, it, x, xarr):
        net.forward(x)
        eng.sync()
        sb = host(net.stats).copy()
        want_z, want_kl = V.latent_fwd(sb, B, L, cls.SEED_LATENT, it + 1)
        assert net.lat.call == it + 1 and np.array_equal(host(net.z).reshape(B, L), want_z)
        assert np.array_equal(net.lat.kl.to_host().view(np.uint32), want_kl.view(np.uint32))
        xb = xarr.to_host().reshape(-1, C_IN)
        g, lw = V.bce_replay(host(net.out), xb, 1, 1.0 / B, target_stride=C_IN)
        assert np.array_equal(host(net.dout).reshape(-1), g.reshape(-1))
        assert np.array_equal(net.loss.cpu().numpy().view(np.uint32), lw.view(np.uint32))
        net.backward()
        eng.sync()
        dzb = host(net.dz)
        assert np.any(dzb != 0)
        assert np.array_equal(host(net.stats).reshape(B, 2 * L), V.latent_bwd(sb, dzb, B, L, cls.SEED_LATENT, it + 1, cls.BETA / B))

    losses, nelbo, rec, kl, base, _ = vae_nets.train_vae(eng, pkg, golden, check_step)
    print(f"ConvVAE: epoch losses {[round(v, 2) for v in losses]}, test negative ELBO {nelbo:.2f} nats (reconstruction {rec:.2f}, "
          f"KL {kl:.2f}; replica {REPLICA_NELBO}), mean-image baseline {base:.2f}")
    assert losses[-1] < losses[0]
    assert nelbo <= base - BASELINE_MARGIN
    assert kl >= KL_FLOOR
    assert abs(nelbo - REPLICA_NELBO) <= NELBO_RTOL * REPLICA_NELBO
