"""Every layer of the five device-trained example networks, on the operands the device actually handed it, across training steps
and in eval (tests/network_tape.py records the calls and holds the checkers).

The networks are the classes of example_nets.py that the end-to-end tests train, run unchanged: the LeNet-style Net, ReluNet,
the BN ResNet, the GAP ResNet and MobileNetLite.  Schedule, on the golden MNIST digits:
- training steps 0 to 3, each followed by the network's own sgd: every checker at steps 0 and 3, the bit-exact ones and the
  batch-norm statistics at steps 1 and 2;
- after the four steps, each batch norm's running mean against running_update chained over the recorded save_mean of every step,
  bit for bit, and its running variance chained the same way, within the bound of test_batchnorm_gpu.test_forward against
  float64 and within fp32 rounding against the device's own batch variance (read back from save_rstd);
- eval (training=False) over every golden test digit, every checker on its own tape;
- a fresh run without the tape gives bit-identical masters and batch-norm state after the same four steps.
Every layer object must appear on the tape in both directions in training and in the forward in eval, and every ReLU output must
be 5-95 % positive, so no check passes for a trivial reason.  The worst ratio of each check to its bound is printed per network
and step, with the count of one-ulp softmax cases.

The tape checks each call against the arguments it was given.  A network class that passes the wrong buffer, or none, at a join
(a dr or dy2 left out) or between layers is outside what it can see: that needs an end-to-end replica of the whole network, which
this file does not have."""
import time

import numpy as np
import pytest
import torch

import batchnorm_ref as BR
import network_tape as NT
from example_nets import DEV, MobileNetLite, Net, ReluNet, ResNet, ResNetGAP, mnist_device

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
NETS = {cls.__name__: cls for cls in (Net, ReluNet, ResNet, ResNetGAP, MobileNetLite)}
STEPS = 4
FULL = (0, STEPS - 1)


def state(net):
    """host copies of every master and batch-norm statistic, as uint32 bit patterns"""
    out = []
    for _, layer in NT.layers_of(net):
        if hasattr(layer, "params"):
            out += [a.view(np.uint32) for a in layer.params() if a is not None]
    return out


class Summary:
    """worst ratio of each check (kind.check) to its bound over the calls of one pass"""

    def __init__(self):
        self.worst, self.calls = {}, []

    def add(self, e, ratios):
        self.calls.append((e["name"], e["op"], e["kind"], e["argv"].get("training")))
        for k, v in ratios.items():
            key = f"{e['kind'].replace('Layer', '')}.{k}"
            self.worst[key] = v + self.worst.get(key, 0) if k == "one-ulp" else max(v, self.worst.get(key, 0.0))

    def line(self):
        return ", ".join(f"{k} {v}" if isinstance(v, int) else f"{k} {v:.3f}" for k, v in sorted(self.worst.items()))


def check_coverage(net, calls, training):
    names = [n for n, _ in NT.layers_of(net)]
    fwd = {n for n, op, _, _ in calls if op == "forward"}
    bwd = {n for n, op, _, _ in calls if op == "backward"}
    assert fwd == set(names), set(names) ^ fwd
    assert sum(op == "softmax" for _, op, _, _ in calls) == 1
    if training:
        assert bwd == set(names), set(names) ^ bwd
    else:
        assert not bwd
    for n, op, kind, tr in calls:
        if kind == "BatchNormLayer" and op == "forward":
            assert tr == training, (n, tr)


def tape_run(eng, pkg, golden, name, net, NB, batch, train, test, n_test):
    """the taped schedule on `net`: STEPS training steps, the running-statistics chains, eval over the n_test test digits;
    returns the masters and batch-norm state after the training steps"""
    xs, ys = train
    xt, yt = test
    bns = [(n, layer) for n, layer in NT.layers_of(net) if type(layer).__name__ == "BatchNormLayer"]
    chain = {n: [] for n, _ in bns}                     # per training step: save_mean, save_rstd, float64 variance, its bound

    def keep_stats(e):
        if "stats" in e:                                # a training batch-norm forward: bn_forward's statistics
            chain[e["name"]].append((e["o"]["save_mean"], e["o"]["save_rstd"], e["stats"]["v64"], e["stats"]["var_bound"]))

    with NT.Tape(eng, net) as tape:
        for step in range(STEPS):
            x, labels, rows = batch(step, xs, ys)
            tape.inputs = {x: rows}
            s = Summary()

            def sink(e, full=step in FULL, s=s):
                r = NT.check(pkg, e, full)
                keep_stats(e)
                s.add(e, r)
            tape.sink = sink
            net.forward(x, labels, training=True)
            net.backward()
            check_coverage(net, s.calls, True)
            print(f"{name} step {step} ({'every check' if step in FULL else 'bit-exact checks'}): {s.line()}")
            net.sgd(net.LR_STEP)
            eng.sync()
        trained = state(net)

        # running statistics chained over the four steps: each call's update is checked on the tape, the chain also catches
        # anything that touches them between calls (sgd, the optimizer) and an update missing or repeated
        for n, L in bns:
            rm_dev, rv_dev = L.running_mean.to_host(), L.running_var.to_host()
            M, mom = L.pixels, L.momentum
            rm = np.zeros(L.shape[3], np.float32)
            rv32 = np.ones(L.shape[3], np.float32)
            want, E, E32 = np.ones(L.shape[3]), np.zeros(L.shape[3]), np.zeros(L.shape[3])
            for mean, rstd, v64, vb in chain[n]:
                rm = BR.running_update(rm, mean, mom)
                want = (1 - mom) * want + mom * v64 * M / (M - 1)
                E = (1 - mom) * E + mom * vb * M / (M - 1) + 4 * U * np.abs(want)
                var_dev = 1.0 / rstd.astype(np.float64) ** 2 - np.float64(np.float32(L.eps))
                unb = (var_dev * M / (M - 1)).astype(np.float32)
                rv32 = BR.running_update(rv32, unb, mom)
                # rstd is fp32-rounded: var + eps from it is off by <= 2.01 u (var + eps), the fp32 quotient by one rounding more;
                # each fp32 running update rounds on both sides
                E32 = (1 - mom) * E32 + mom * (2.01 * U * (var_dev + L.eps) * M / (M - 1) + 2 * U * np.abs(unb)) + 4 * U * np.abs(rv32)
            assert len(chain[n]) == STEPS
            assert np.array_equal(rm_dev.view(np.uint32), rm.view(np.uint32)), n
            r64 = float(np.max(np.abs(rv_dev - want) / E))
            r32 = float(np.max(np.abs(rv_dev.astype(np.float64) - rv32) / (E32 + 1e-30)))
            print(f"{name} {n}: running_var vs float64 chain {r64:.3f} of its bound, vs the device's batch variance {r32:.3f}")
            assert r64 <= 1 and r32 <= 1, (n, r64, r32)

        right, s = 0, Summary()
        for b in range(n_test // NB):                     # eval over every golden test digit
            x, labels, rows = batch(b, xt, yt)
            tape.inputs = {x: rows}
            sb = Summary()

            def sink(e, sb=sb):
                r = NT.check(pkg, e, True)
                sb.add(e, r)
                s.add(e, r)
            tape.sink = sink
            net.forward(x, labels, training=False)
            check_coverage(net, sb.calls, False)
            right += int((net.pred.cpu().numpy() == golden["test_labels"][b * NB:(b + 1) * NB]).sum())
        print(f"{name} eval (accuracy {right / n_test:.4f} after {STEPS} steps): {s.line()}")
    assert all(np.array_equal(a, b) for a, b in zip(state(net), trained))         # eval changed nothing
    return trained


@pytest.mark.parametrize("name", list(NETS))
def test_network_tape(eng, pkg, golden, name):
    t0 = time.time()
    cls = NETS[name]
    NB = cls.NB
    xs, ys = mnist_device(pkg, golden["train_u8"]), torch.from_numpy(golden["train_labels"]).to(DEV)
    xt, yt = mnist_device(pkg, golden["test_u8"]), torch.from_numpy(golden["test_labels"]).to(DEV)

    def batch(s, xs, ys):
        rows = xs[s * NB * 28:(s + 1) * NB * 28]
        return rows.data_ptr(), ys[s * NB:(s + 1) * NB], rows

    n_test = len(golden["test_labels"])
    assert n_test % NB == 0, (n_test, NB)
    net = cls(eng, pkg, cls.init_params())
    try:
        trained = tape_run(eng, pkg, golden, name, net, NB, batch, (xs, ys), (xt, yt), n_test)
    finally:
        net.close()

    fresh = cls(eng, pkg, cls.init_params())              # the tape is harmless: the same steps without it
    try:
        for step in range(STEPS):
            x, labels, _ = batch(step, xs, ys)
            fresh.forward(x, labels, training=True)
            fresh.backward()
            fresh.sgd(cls.LR_STEP)
        eng.sync()
        again = state(fresh)
    finally:
        fresh.close()
    assert len(again) == len(trained) and all(np.array_equal(a, b) for a, b in zip(again, trained))
    print(f"{name}: {time.time() - t0:.1f} s")
