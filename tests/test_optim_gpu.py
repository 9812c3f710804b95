"""The fused optimizers on the device (pcnn_optim_*, FusedOptimizer, SGD, AdamW): params and state bit-identical to the float32 replays
of tests/optim_ref.py (pinned to torch.optim by test_optim_cpu.py) on special values, on both the vector and the scalar path and on a
ResNet-18-sized table with several chunks per CTA; the plans' operands refreshed to exactly what a plan created from the new masters
holds; momentum 0 without decay bit-identical to the layers' own sgd(lr) on the GAP ResNet; that network trained with momentum SGD
and with AdamW; every refusal."""
import numpy as np
import pytest
import torch

import optim_ref as R
from example_nets import DEV, ResNetGAP, Slices, host, same_bits, train

pytestmark = pytest.mark.gpu



def same(got, want):
    """float32 arrays: NaN where want is NaN (any payload), the same bits everywhere else"""
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))


def special(rng, n, scale=1.0):
    """normal values with +-0, subnormals, +-Inf and NaN sprinkled in"""
    x = (rng.standard_normal(n) * scale).astype(np.float32)
    k = max(1, n // 20)
    for v in (0.0, -0.0, np.inf, -np.inf, np.nan, 1e-40, -3e-39, 1e-45):
        x[rng.choice(n, min(n, k), replace=False)] = v
    return x


class RawTable:
    """tensors of sizes `sizes` in one param and one grad buffer, each starting on a 256-byte boundary plus `offsets[i]` floats (1 puts
    it on the scalar path)"""

    def __init__(self, eng, sizes, offsets):
        self.sizes, self.starts = sizes, []
        at = 0
        for n, o in zip(sizes, offsets):
            at = (at + 63) // 64 * 64 + o
            self.starts.append(at)
            at += n
        self.total = at
        self.p, self.g = eng.array(self.total), eng.array(self.total)
        self.ph, self.gh = np.zeros(self.total, np.float32), np.zeros(self.total, np.float32)

    def views(self, a):
        return [a[s:s + n] for s, n in zip(self.starts, self.sizes)]

    def tensors(self, wds):
        return [(self.p.ptr + 4 * s, self.g.ptr + 4 * s, n, wd, None, 0) for s, n, wd in zip(self.starts, self.sizes, wds)]

    def set(self, params=None, grads=None):
        if params is not None:
            for v, x in zip(self.views(self.ph), params):
                v[:] = x
            self.p.copy_from(self.ph)
        if grads is not None:
            for v, x in zip(self.views(self.gh), grads):
                v[:] = x
            self.g.copy_from(self.gh)

    def params(self):
        return [v.copy() for v in self.views(self.p.to_host())]


CONFIGS = [("sgd", dict(momentum=0.0)), ("sgd-momentum-dampening", dict(momentum=0.9, dampening=0.1)),
           ("sgd-nesterov", dict(momentum=0.9, nesterov=True)), ("adamw", dict(betas=(0.9, 0.999), eps=1e-8)),
           ("adamw-b0.5", dict(betas=(0.5, 0.9), eps=1e-3))]


def make_opt(pkg, eng, name, kw, tensors):
    kind = pkg.OPTIM_ADAMW if name.startswith("adamw") else pkg.OPTIM_SGD
    return pkg.FusedOptimizer(eng, kind, tensors, **kw)


def replay(name, kw, p, g, s0, s1, lr, t, wd):
    if name.startswith("adamw"):
        b1, b2 = kw["betas"]
        return R.adamw32(p, g, s0, s1, lr, t, b1, b2, kw["eps"], wd)
    p, b = R.sgd32(p, g, s0, lr, t, kw.get("momentum", 0.0), kw.get("dampening", 0.0), kw.get("nesterov", False), wd)
    return p, b, None


def run_table(pkg, eng, name, kw, table, p0, grads_by_step, lrs, wds, check=True):
    """steps over a RawTable; after each step params and state are compared with the replay.  Returns the final params"""
    table.set(params=p0)
    opt = make_opt(pkg, eng, name, kw, table.tensors(wds))
    ps = [p.copy() for p in p0]
    st = [(None, None)] * len(ps)
    if name.startswith("adamw"):
        st = [(np.zeros_like(p), np.zeros_like(p)) for p in ps]
    for t, (gs, lr) in enumerate(zip(grads_by_step, lrs), 1):
        table.set(grads=gs)
        opt.step(lr)
        eng.sync()
        if not check:
            continue
        got, got_state = table.params(), opt.state()
        for i in range(len(ps)):
            p, s0, s1 = replay(name, kw, ps[i], gs[i], st[i][0], st[i][1], lr, t, wds[i])
            ps[i], st[i] = p, (s0, s1)
            assert same(got[i], p), (name, t, i, int(np.sum(got[i].view(np.uint32) != p.view(np.uint32))))
            for a, b in zip(got_state[i], (s0, s1)):
                assert (a is None) == (b is None) and (a is None or same(a, b)), (name, t, i, "state")
    assert opt.steps == len(lrs)
    info = opt.info()
    opt.close()
    return table.params(), info


NS = [1, 3, 4, 7, 1000, 4099, (1 << 20) + 3, 65536]


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_bit_exact_update(eng, pkg, cfg):
    name, kw = cfg
    sizes = NS + NS
    offsets = [0] * len(NS) + [1] * len(NS)
    wds = [1e-2 if i % 2 else 0.0 for i in range(len(sizes))]
    rng = np.random.default_rng(7)
    table = RawTable(eng, sizes, offsets)
    p0 = [special(rng, n) for n in sizes]
    grads = [[special(rng, n, 0.1) for n in sizes] for _ in range(5)]
    lrs = [0.1, 0.05, 0.2, 0.01, 0.3] if name.startswith("sgd") else [1e-3, 3e-3, 2e-3, 5e-4, 1e-2]
    final, info = run_table(pkg, eng, name, kw, table, p0, grads, lrs, wds)
    vec = sum(1 for n, o in zip(sizes, offsets) if n % 4 == 0 and o == 0)
    assert info["tensors"] == len(sizes) and info["elements"] == sum(sizes) and info["vector_tensors"] == vec
    assert info["chunks"] == sum((n + 4095) // 4096 for n in sizes)
    again, _ = run_table(pkg, eng, name, kw, table, p0, grads, lrs, wds, check=False)            # rerun
    assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(final, again))


@pytest.mark.parametrize("name,kw", [("sgd-momentum", dict(momentum=0.9)), ("adamw", dict(betas=(0.9, 0.999), eps=1e-8))])
def test_resnet18_table_many_chunks_per_cta(eng, pkg, name, kw):
    tensors = R.resnet18_tensors()
    sizes = [int(np.prod(s)) for _, s, _ in tensors]
    wds = [0.0 if len(s) == 1 else 5e-4 for _, s, _ in tensors]
    rng = np.random.default_rng(18)
    table = RawTable(eng, sizes, [0] * len(sizes))
    p0 = [(rng.standard_normal(n) * 0.05).astype(np.float32) for n in sizes]
    grads = [[(rng.standard_normal(n) * 1e-2).astype(np.float32) for n in sizes] for _ in range(2)]
    _, info = run_table(pkg, eng, name, kw, table, p0, grads, [0.1, 0.05] if name.startswith("sgd") else [1e-3, 2e-3], wds)
    sm = eng.device_info()["sm_count"]
    assert len(sizes) == 62 and info["elements"] == 11_689_512 and info["vector_tensors"] == 62
    assert info["grid"] <= 4 * sm and info["chunks"] > 2 * info["grid"], (info, sm)
    print(f"ResNet-18 table ({name}): {info['chunks']} chunks over a grid of {info['grid']} ({sm} SMs): "
          f"{info['chunks'] / info['grid']:.2f} chunks per CTA")


# ------------------------------------------------------------------------------------------------ plan refresh
def bf16_input(pkg, rng, shape):
    return torch.from_numpy(pkg.f32_to_bf16_bits(rng.standard_normal(shape).astype(np.float32)).view(np.int16)).to(DEV)


def make_layers(pkg, eng, params):
    """the plans of the refresh test from host parameters: row-Toeplitz LeNet c1 (K = 6) and a V = 2 shape, wide "same", stride 2 and
    C = 320, linear with Q*C = 9 (a pitch with pad) and O = 10, with and without bias"""
    relu = pkg.ACT_RELU
    C_ = pkg.ConvLayer
    return [C_(eng, 2, 28, 28, 1, 6, 5, 5, params[0][0], params[0][1], act=relu),
            C_(eng, 2, 12, 12, 3, 8, 5, 5, params[1][0], params[1][1], act=relu),
            C_(eng, 2, 12, 12, 16, 16, 3, 3, params[2][0], params[2][1], act=relu, padding=(1, 1)),
            C_(eng, 2, 12, 12, 16, 32, 3, 3, params[3][0], params[3][1], act=relu, stride=2, padding=(1, 1)),
            C_(eng, 2, 6, 6, 320, 16, 3, 3, params[4][0], params[4][1], act=relu, padding=(1, 1)),
            pkg.LinearLayer(eng, 4, 3, 3, 3, 10, params[5][0], params[5][1], act=relu),
            pkg.LinearLayer(eng, 4, 3, 3, 3, 10, params[6][0], None)]


SHAPES = [((6, 5, 5, 1), 6), ((8, 5, 5, 3), 8), ((16, 3, 3, 16), 16), ((32, 3, 3, 16), 32), ((16, 3, 3, 320), 16), ((10, 3, 3, 3), 10),
          ((10, 3, 3, 3), None)]


def layer_io(pkg, rng, layer):
    if isinstance(layer, pkg.LinearLayer):
        N, P, Q, C, O = layer.shape
        return bf16_input(pkg, rng, (N, P, layer.row_pitch)), (N, O)
    N, H, W, C, K, R_, S = layer.shape
    return bf16_input(pkg, rng, (N, H, layer.row_pitch)), layer.out_shape


def buffers(pkg, layers, xs, ys):
    """output buffers of one pass over the layers: y, and dx for a linear layer (allocated before any engine work reads them)"""
    out = [[torch.zeros(y, dtype=torch.int16, device=DEV)] + ([torch.zeros_like(x)] if isinstance(layer, pkg.LinearLayer) else [])
           for layer, x, y in zip(layers, xs, ys)]
    torch.cuda.synchronize()
    return out


def run_outputs(pkg, eng, layers, xs, dys, bufs):
    """the forward (and for a linear layer the input gradient) of every layer with its plan, enqueued on the engine's stream"""
    for layer, x, dy, b in zip(layers, xs, dys, bufs):
        layer.forward(x, b[0])
        if isinstance(layer, pkg.LinearLayer):
            eng.linear_dgrad(layer.plan, dy, b[1])


def bits(bufs):
    return [[host(t) for t in b] for b in bufs]


@pytest.mark.parametrize("kind", ["sgd", "adamw"])
def test_plan_refresh(eng, pkg, kind):
    rng = np.random.default_rng(33)
    params = [(rng.uniform(-0.3, 0.3, s).astype(np.float32), None if k is None else rng.uniform(-0.3, 0.3, k).astype(np.float32))
              for s, k in SHAPES]
    lr = 0.05 if kind == "sgd" else 1e-2

    def build():
        layers = make_layers(pkg, eng, params)
        opt = (pkg.SGD(eng, layers, momentum=0.9, weight_decay=1e-2, decay_norm_and_bias=False) if kind == "sgd"
               else pkg.AdamW(eng, layers, weight_decay=1e-2))
        for layer, (gw, gb) in zip(layers, grads):
            layer.dw.copy_from(gw)
            if gb is not None:
                layer.db.copy_from(gb)
        return layers, opt

    probe = make_layers(pkg, eng, params)
    assert [layer.family for layer in probe[:5]] == ["narrow", "narrow", "wide", "wide", "wide"]
    xs, ys = zip(*(layer_io(pkg, rng, layer) for layer in probe))
    dys = [bf16_input(pkg, rng, y) if isinstance(layer, pkg.LinearLayer) else None for layer, y in zip(probe, ys)]
    grads = [(rng.standard_normal(layer.dw.shape).astype(np.float32), None if layer.db is None else rng.standard_normal(layer.db.shape).astype(np.float32))
             for layer in probe]
    for layer in probe:
        layer.close()

    # synchronised: after each step the outputs equal those of plans created afresh from the new host masters
    layers, opt = build()
    synced = []
    for it in range(3):
        b = buffers(pkg, layers, xs, ys)
        run_outputs(pkg, eng, layers, xs, dys, b)
        eng.sync()
        synced.append(bits(b))
        if it:
            fresh = make_layers(pkg, eng, [layer.params() for layer in layers])
            fb = buffers(pkg, fresh, xs, ys)
            run_outputs(pkg, eng, fresh, xs, dys, fb)
            eng.sync()
            for i, (g, w) in enumerate(zip(synced[-1], bits(fb))):
                assert all(np.array_equal(x, y) for x, y in zip(g, w)), (kind, it, i)
            for layer in fresh:
                layer.close()
        opt.step(lr)
        eng.sync()
    opt.close()
    for layer in layers:
        layer.close()

    # interleaved forward -> step -> forward with no synchronisation in between: the same outputs
    layers, opt = build()
    bufs = [buffers(pkg, layers, xs, ys) for _ in range(3)]
    for it in range(3):
        run_outputs(pkg, eng, layers, xs, dys, bufs[it])
        opt.step(lr)
    eng.sync()
    for it in range(3):
        for i, (g, w) in enumerate(zip(bits(bufs[it]), synced[it])):
            assert all(np.array_equal(x, y) for x, y in zip(g, w)), (kind, "interleaved", it, i)
    opt.close()
    for layer in layers:
        layer.close()


# ------------------------------------------------------------------------------------------------ the GAP ResNet
def test_momentum0_matches_layer_sgd(eng, pkg, golden):
    """SGD with momentum 0 and no decay gives the bits of every layer's sgd(lr): params, running statistics and logits"""
    slices = Slices(pkg, golden["train_u8"], golden["train_labels"], ResNetGAP.NB)
    a, b = ResNetGAP(eng, pkg, ResNetGAP.init_params()), ResNetGAP(eng, pkg, ResNetGAP.init_params())
    torch.cuda.synchronize()
    opt = pkg.SGD(eng, b.layers())
    launches = []
    for it in range(5):
        for net in (a, b):
            net.forward(*slices.batch(it))
            net.backward()
        a.sgd(0.2)
        n0 = eng.launch_count()
        opt.step(0.2)
        launches.append(eng.launch_count() - n0)
        eng.sync()
        assert np.array_equal(host(a.z), host(b.z)), it
        assert same_bits(a.params(), b.params()), it
    assert launches == [2] * 5                         # the update and c1's Toeplitz gather
    opt.close()
    a.close()
    b.close()


EPOCHS = 40
E2E = {  # kind: (optimizer kwargs, lr, threshold); a float32 torch CPU replica with torch.optim reaches 0.953 / 0.957 (DESIGN 3.17)
    "sgd": (dict(momentum=0.9, weight_decay=5e-4), 0.02, 0.88),
    "adamw": (dict(betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2), 1e-3, 0.88),
}


@pytest.mark.parametrize("kind", list(E2E))
def test_resnet_gap_trains(eng, pkg, golden, kind):
    """In each of the first 5 steps the masters after the step are bit-exact against the replay on the device's own gradients; a fresh
    run reproduces them.  After EPOCHS epochs the test accuracy with the running statistics exceeds the threshold."""
    kw, lr, acc_min = E2E[kind]
    Opt = pkg.SGD if kind == "sgd" else pkg.AdamW

    class Optimized(ResNetGAP):
        """the GAP ResNet with its own fused optimizer over every layer"""

        def __init__(self):
            super().__init__(eng, pkg, ResNetGAP.init_params())
            torch.cuda.synchronize()
            self.opt = Opt(eng, self.layers(), **kw)

        def close(self):
            self.opt.close()
            super().close()

    before = {}                                         # the step's operands, from check_step to update

    def check_step(net, it, x, labels):
        net.forward(x, labels)
        net.backward()
        eng.sync()
        tab = [t for layer in net.layers() for t in layer.optim_tensors()]
        before.update(it=it, tab=tab, ps=[p.to_host().ravel() for p, *_ in tab], gs=[g.to_host().ravel() for _, g, *_ in tab],
                      state=net.opt.state())

    def update(net):
        net.opt.step(lr)
        if before:
            eng.sync()
            it, tab, state, wd = before["it"], before["tab"], before["state"], kw["weight_decay"]
            for i, (p, g) in enumerate(zip(before["ps"], before["gs"])):
                if kind == "sgd":
                    want, _ = R.sgd32(p, g, state[i][0], lr, it + 1, kw["momentum"], 0.0, False, wd)
                else:
                    want, _, _ = R.adamw32(p, g, state[i][0], state[i][1], lr, it + 1, *kw["betas"], kw["eps"], wd)
                assert same(tab[i][0].to_host().ravel(), want), (kind, it, i)
            before.clear()

    def check_trained(net):
        assert net.opt.steps == EPOCHS * 8

    ep_loss, acc, _ = train(eng, pkg, golden, Optimized, EPOCHS, update=update, check_step=check_step, check_trained=check_trained)
    print(f"GAP ResNet with {kind} lr {lr}: mean loss by epoch {ep_loss[0]:.4f} -> {ep_loss[-1]:.4f}; test accuracy {acc:.4f} (threshold {acc_min})")
    assert np.isfinite(ep_loss).all() and ep_loss[-1] < ep_loss[0]
    assert acc > acc_min


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(eng, pkg):
    p, g, q = eng.array(64), eng.array(64), eng.array(64)
    conv = pkg.ConvLayer(eng, 2, 12, 12, 16, 16, 3, 3, np.zeros((16, 3, 3, 16), np.float32), None, padding=(1, 1))
    fc = pkg.LinearLayer(eng, 4, 1, 1, 8, 10, np.zeros((10, 8), np.float32), np.zeros(10, np.float32))
    SGD, ADAMW = pkg.OPTIM_SGD, pkg.OPTIM_ADAMW
    T = lambda *rows: list(rows)
    ok = (p, g, 64, 0.0, None, 0)
    cases = [
        (SGD, T(), {}, "pcnn_optim_create: count 0 < 1"),
        (SGD, T((None, g, 64, 0.0, None, 0)), {}, "tensor 0: NULL param or grad"),
        (SGD, T((p, None, 64, 0.0, None, 0)), {}, "tensor 0: NULL param or grad"),
        (SGD, T((p, g, 0, 0.0, None, 0)), {}, "tensor 0: n = 0 <= 0"),
        (SGD, T(ok, (p.ptr + 64, q, 8, 0.0, None, 0)), {}, "overlapping buffers: the param of tensor 0 and the param of tensor 1"),
        (SGD, T((p, p, 64, 0.0, None, 0)), {}, "overlapping buffers"),
        (SGD, T(ok, (q, g.ptr + 128, 8, 0.0, None, 0)), {}, "overlapping buffers: the grad of tensor 0 and the grad of tensor 1"),
        (SGD, T((conv.filt, conv.dw, 100, 0.0, conv.plan, 1)), {}, "n = 100, but the plan's filters / weights have 2304 elements"),
        (SGD, T((fc.w, fc.dw, 81, 0.0, fc.plan, 1)), {}, "n = 81, but the plan's filters / weights have 80 elements"),
        (SGD, T((fc.bias, fc.db, 8, 0.0, fc.plan, 2)), {}, "n = 8, but the plan's bias has 10 elements"),
        (SGD, T((p, g, 16, 0.0, conv.plan, 2)), {}, "a bias for a plan created without one"),
        (SGD, T((fc.w, fc.dw, 80, 0.0, fc.plan, 1), (p, g, 80 // 2, 0.0, fc.plan, 1)), {}, "the same plan part \\(1\\) listed twice"),
        (SGD, T((p, g, 64, 0.0, None, 3)), {}, "plan_part 3 is not 0"),
        (SGD, T((p, g, 64, 0.0, None, 1)), {}, "plan_part 1 without a plan"),
        (SGD, T((p, g, 64, 0.0, fc.plan, 0)), {}, "plan_part 0 with a plan"),
        (2, T(ok), {}, "kind 2 is not PCNN_OPTIM_SGD"),
        (SGD, T(ok), dict(momentum=-0.1), "momentum -0.1 < 0"),
        (SGD, T(ok), dict(momentum=float("nan")), "momentum or dampening is NaN"),
        (SGD, T(ok), dict(dampening=float("nan")), "momentum or dampening is NaN"),
        (SGD, T(ok), dict(nesterov=True), "nesterov needs momentum > 0 and dampening 0"),
        (SGD, T(ok), dict(nesterov=True, momentum=0.9, dampening=0.1), "nesterov needs momentum > 0 and dampening 0"),
        (ADAMW, T(ok), dict(betas=(1.0, 0.999)), "betas \\(1, 0.999\\) outside \\[0, 1\\)"),
        (ADAMW, T(ok), dict(betas=(0.9, -0.5)), "outside \\[0, 1\\)"),
        (ADAMW, T(ok), dict(betas=(float("nan"), 0.9)), "beta1, beta2 or eps is NaN"),
        (ADAMW, T(ok), dict(eps=-1e-8), "eps -1e-08 < 0"),
        (ADAMW, T(ok), dict(eps=float("nan")), "beta1, beta2 or eps is NaN"),
        (SGD, T((p, g, 64, -0.01, None, 0)), {}, "tensor 0: weight_decay -0.01 < 0"),
        (ADAMW, T((p, g, 64, float("nan"), None, 0)), {}, "tensor 0: weight_decay is NaN"),
    ]
    for kind, tensors, kw, msg in cases:
        with pytest.raises(pkg.PcnnError, match=msg):
            pkg.FusedOptimizer(eng, kind, tensors, **kw)
    opt = pkg.FusedOptimizer(eng, SGD, [ok])
    for lr, msg in ((-0.1, "pcnn_optim_step: lr -0.1: must be >= 0 and not NaN"), (float("nan"), "lr nan: must be >= 0 and not NaN")):
        with pytest.raises(pkg.PcnnError, match=msg):
            opt.step(lr)
    assert opt.steps == 0
    opt.step(0.1)
    eng.sync()
    assert opt.steps == 1
    opt.close()
    conv.close()
    fc.close()
