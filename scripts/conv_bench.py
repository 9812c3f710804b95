#!/usr/bin/env python
"""scripts/conv_bench.py -- throughput of the bf16 wgmma convolution forward (BASELINE.json configs 3 and 5) against the
HBM roofline.  Algorithmic bytes per image are SURVEY.md 8d's: each operand crosses HBM once (input read + output written,
bf16): LeNet c1 8,480 B, 224x224x3 -> 64 x 3x3: 6,609,408 B.  CUDA-event timing over back-to-back launches after warm-up;
the working set of every measured point except the smallest batches exceeds the 50 MB L2."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pcnn_loader  # noqa: E402

pkg = pcnn_loader.load()
torch.cuda.set_device(0)
stream = torch.cuda.Stream()
torch.cuda.set_stream(stream)
eng = pkg.Engine(0, stream.cuda_stream)
HBM = 3350.0                        # GB/s, NVIDIA H100 SXM data sheet (HBM3)
rng = np.random.default_rng(1234)
only = sys.argv[1] if len(sys.argv) > 1 else "all"


def run(name, N, H, W, C, K, R, S, act, iters, image_rows=0, bias=True):
    pitch = (W * C + 7) // 8 * 8
    P, Q = H - R + 1, W - S + 1
    f = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    plan = pkg.ConvPlan(eng, N, H, W, C, K, R, S, f, b if bias else None, act=act, row_pitch=pitch, image_rows=image_rows)
    x = torch.randint(0, 0x3F80, (N * (image_rows or H), pitch), dtype=torch.int16, device="cuda")   # positive bf16 bit patterns < 1.0
    y = torch.empty((N, P, Q, K), dtype=torch.int16, device="cuda")
    for _ in range(3):
        plan.fwd(x, y)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(iters):
        plan.fwd(x, y)
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    alg = N * (H * W * C + P * Q * K) * 2                       # bf16 in + out, once each
    flops = 2.0 * N * P * Q * K * R * S * C
    row = {"case": name, "N": N, "ms": ms, "img_per_s": N / (ms * 1e-3), "alg_GBps": alg / (ms * 1e-3) / 1e9,
           "hbm_frac": alg / (ms * 1e-3) / 1e9 / HBM, "useful_TFLOPs": flops / (ms * 1e-3) / 1e12,
           "working_set_MB": (N * H * pitch + N * P * Q * K) * 2 / 1e6}
    print(json.dumps(row), flush=True)
    plan.close()
    del x, y


def run_bwd(name, N, H, W, C, K, R, S, iters, stride=1):
    """wgrad and dgrad of the same layer: algorithmic bytes = dy read + x read (wgrad) / dy read + dx written (dgrad), bf16."""
    P, Q = (H - R) // stride + 1, (W - S) // stride + 1
    xb = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    dyb = torch.randint(0, 0x3F80, (N, P, Q, K), dtype=torch.int16, device="cuda")
    dyb ^= (torch.randint(0, 2, (N, P, Q, K), dtype=torch.int16, device="cuda") << 15)      # random signs
    f = torch.rand((K, R, S, C), dtype=torch.float32, device="cuda") - 0.5
    dw = torch.empty((K, R, S, C), dtype=torch.float32, device="cuda")
    dx = torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    alg = N * (H * W * C + P * Q * K) * 2
    flops = 2.0 * N * P * Q * K * R * S * C
    for what, fn in (("wgrad", lambda: eng.conv_wgrad(xb, dyb, dw, N, H, W, C, K, R, S, stride=stride)),
                     ("dgrad", lambda: eng.conv_dgrad(dyb, f, dx, N, H, W, C, K, R, S, stride=stride))):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        import time
        e0.record(stream)
        t0 = time.perf_counter()
        for _ in range(iters):
            fn()
        host_us = (time.perf_counter() - t0) / iters * 1e6           # host time to enqueue one call
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        print(json.dumps({"case": name + " " + what, "host_enqueue_us": host_us, "N": N, "ms": ms, "img_per_s": N / (ms * 1e-3), "alg_GBps": alg / (ms * 1e-3) / 1e9,
                          "hbm_frac": alg / (ms * 1e-3) / 1e9 / HBM, "useful_TFLOPs": flops / (ms * 1e-3) / 1e12, "stride": stride,
                          "path": os.environ.get("PCNN_CONV_BWD", "tc"), "working_set_MB": alg / 1e6}), flush=True)
    del xb, dyb, dx


def card():
    """name and power limit of GPU 0, read (never set) in the same run as the measurement"""
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power = [t.strip() for t in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def _bf(shape, scale=1.0):
    return (torch.randn(shape, device="cuda") * scale).to(torch.bfloat16)


def _line(case, ms, ms_torch, nbytes=None, **extra):
    gpu, power = card()
    d = {"case": case, "us": ms * 1e3, "torch_us": ms_torch * 1e3, "torch_over_ours": ms_torch / ms, "gpu": gpu, "power_limit": power}
    if nbytes:
        d.update(MB=nbytes / 1e6, hbm_frac=nbytes / (ms * 1e-3) / 1e9 / HBM)
    d.update(extra)
    print(json.dumps(d), flush=True)


def run_convt(name, N, H, W, Ci, Co, R, stride, pad, iters, rounds=3):
    """ConvTransposeLayer forward and backward (dx and dw) against torch eager conv_transpose2d and its autograd, on the same bf16
    channels-last tensors; FLOPs 2 N H W Ci Co R R per pass"""
    w = (np.random.default_rng(0).standard_normal((Ci, Co, R, R)) / np.sqrt(Ci * R * R)).astype(np.float32)
    layer = pkg.ConvTransposeLayer(eng, N, H, W, Ci, Co, R, R, w, stride=stride, padding=(pad, pad))
    _, Ho, Wo, _ = layer.out_shape
    x, dy = _bf((N, H, W, Ci)), _bf((N, Ho, Wo, Co))
    y, dx = torch.empty((N, Ho, Wo, Co), dtype=torch.bfloat16, device="cuda"), torch.empty_like(x)
    xt = x.permute(0, 3, 1, 2).requires_grad_(True)
    wt = torch.from_numpy(w).to("cuda", torch.bfloat16).requires_grad_(True)
    dyt = dy.permute(0, 3, 1, 2)
    F = torch.nn.functional
    ours = {"fwd": lambda: layer.forward(x, y), "bwd": lambda: layer.backward(y, dy, dx)}
    theirs = {"fwd": lambda: F.conv_transpose2d(xt, wt, stride=stride, padding=pad),
              "bwd": lambda: torch.autograd.grad(F.conv_transpose2d(xt, wt, stride=stride, padding=pad), (xt, wt), dyt)}
    flops = 2.0 * N * H * W * Ci * Co * R * R
    best = {}
    for _ in range(rounds):
        for k in ours:
            a, b = timed(ours[k], iters), timed(theirs[k], iters)
            o = best.get(k, (a, b))
            best[k] = (min(a, o[0]), min(b, o[1]))
    for k, (a, b) in best.items():
        f = flops * (1 if k == "fwd" else 2)
        _line(f"convt {name} {k}" + (" (torch: fwd + bwd)" if k == "bwd" else ""), a, b, N=N, TFLOPs=f / (a * 1e-3) / 1e12,
              bf16_peak_frac=f / (a * 1e-3) / 1e12 / 989.0)
    layer.close()


def run_upsample(name, N, H, W, C, f, iters, rounds=3):
    """bilinear x f forward and backward against torch interpolate and its autograd (channels-last bf16); bytes: x + y each way"""
    Ho, Wo = H * f, W * f
    layer = pkg.UpsampleBilinearLayer(eng, N, H, W, C, Ho, Wo)
    x, dy = _bf((N, H, W, C)), _bf((N, Ho, Wo, C))
    y, dx = torch.empty_like(dy), torch.empty_like(x)
    xt = x.permute(0, 3, 1, 2).requires_grad_(True)
    dyt = dy.permute(0, 3, 1, 2)
    F = torch.nn.functional
    up = lambda: F.interpolate(xt, size=(Ho, Wo), mode="bilinear", align_corners=False)
    yt = up()
    ours = {"fwd": lambda: layer.forward(x, y), "bwd": lambda: layer.backward(dy, dx)}
    theirs = {"fwd": up, "bwd": lambda: torch.autograd.grad(yt, xt, dyt, retain_graph=True)}
    nbytes = 2 * N * C * (H * W + Ho * Wo)
    best = {}
    for _ in range(rounds):
        for k in ours:
            a, b = timed(ours[k], iters), timed(theirs[k], iters)
            o = best.get(k, (a, b))
            best[k] = (min(a, o[0]), min(b, o[1]))
    for k, (a, b) in best.items():
        _line(f"upsample {name} x{f} {k}", a, b, nbytes, N=N)


def run_segce(N, O, iters, rounds=3):
    """per-pixel CE with ignore index 255 (about 10 % ignored) against torch cross_entropy(ignore_index=255) forward + backward"""
    P = N * 224 * 224
    z = _bf((P, O), 3.0)
    t = torch.randint(0, O, (P,), dtype=torch.uint8, device="cuda")
    t[torch.rand(P, device="cuda") < 0.1] = 255
    d = torch.empty_like(z)
    loss = torch.empty(P, dtype=torch.float32, device="cuda")
    pred = torch.empty(P, dtype=torch.int32, device="cuda")
    cnt = torch.empty(1, dtype=torch.int32, device="cuda")
    zt = z.clone().requires_grad_(True)
    tl = t.long()
    F = torch.nn.functional
    ours = lambda: eng.softmax_ce_pixels_bf16(z, t, P, O, 255, d, cnt, loss, pred)
    theirs = lambda: torch.autograd.grad(F.cross_entropy(zt, tl, ignore_index=255), zt)
    best = None
    for _ in range(rounds):
        a, b = timed(ours, iters), timed(theirs, iters)
        best = (a, b) if best is None else (min(a, best[0]), min(b, best[1]))
    _line(f"segce {P} pixels x {O} classes", best[0], best[1], P * (4 * O + 1 + 8), pixels=P)


def run_fcn(iters):
    """one FCNLite training step (forward, backward, SGD with momentum) at N = 32 on 28 x 28 digits"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import segment_nets
    import segment_ref
    d = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    cls = segment_nets.FCNLite
    net = cls(eng, pkg, cls.init_params())
    opt = pkg.SGD(eng, net.layers(), momentum=0.9)
    b = pkg.ImageBatcher(eng, d["train_u8"].reshape(-1, 28, 28), d["train_labels"], cls.NB, pad=2, flip=True, C_out=8,
                         masks=segment_ref.digit_masks(d["train_u8"], d["train_labels"]))
    def step():
        net.forward(*b.batch(0))
        net.backward()
        opt.step(cls.LR)
    ms = timed(step, iters)
    gpu, power = card()
    print(json.dumps({"case": f"FCNLite training step N={cls.NB}", "us": ms * 1e3, "gpu": gpu, "power_limit": power}), flush=True)
    b.close()
    opt.close()
    net.close()


def run_pixelshuffle(name, N, H, W, C, r, iters, rounds=3):
    """pixel shuffle of x [N][H][W][C r^2] -> [N][H r][W r][C] and the unshuffle of that fine map back, against F.pixel_shuffle /
    F.pixel_unshuffle on the same channels-last bf16 tensors; bytes: each map read or written once"""
    x, fine = _bf((N, H, W, C * r * r)), _bf((N, H * r, W * r, C))
    y, u = torch.empty_like(fine), torch.empty_like(x)
    xt, ft = x.permute(0, 3, 1, 2), fine.permute(0, 3, 1, 2)
    F = torch.nn.functional
    info = pkg.pixel_shuffle_info(N, H, W, C, r)
    ours = {"shuffle": lambda: eng.pixel_shuffle(x, y, N, H, W, C, r), "unshuffle": lambda: eng.pixel_unshuffle(fine, u, N, H * r, W * r, C, r)}
    theirs = {"shuffle": lambda: F.pixel_shuffle(xt, r), "unshuffle": lambda: F.pixel_unshuffle(ft, r)}
    best = {}
    for _ in range(rounds):
        for k in ours:
            a, b = timed(ours[k], iters), timed(theirs[k], iters)
            o = best.get(k, (a, b))
            best[k] = (min(a, o[0]), min(b, o[1]))
    for k, (a, b) in best.items():
        _line(f"pixel {k} {name} r{r}", a, b, 2 * 2 * x.numel(), N=N, path="16-byte" if info["vec"] == 8 else "scalar")


def run_regloss(name, N, H, W, C, iters, rounds=3):
    """the regression loss (dpred and the per-pixel loss) in both modes against torch's mse_loss / l1_loss forward plus autograd
    backward on the same bf16 tensors; bytes: pred and target read, dpred written (bf16), the loss written (fp32)"""
    P = N * H * W
    pred, target = _bf((P, C)), _bf((P, C))
    d, loss = torch.empty_like(pred), torch.empty(P, dtype=torch.float32, device="cuda")
    pt = pred.clone().requires_grad_(True)
    F = torch.nn.functional
    for mode, fn in ((pkg.LOSS_MSE, F.mse_loss), (pkg.LOSS_L1, F.l1_loss)):
        ours = lambda: eng.regression_loss_bf16(pred, target, P, C, d, loss, mode=mode)
        theirs = lambda: torch.autograd.grad(fn(pt, target), pt)
        best = None
        for _ in range(rounds):
            a, b = timed(ours, iters), timed(theirs, iters)
            best = (a, b) if best is None else (min(a, best[0]), min(b, best[1]))
        _line(f"regloss {name} {'mse' if mode == pkg.LOSS_MSE else 'l1'}", best[0], best[1], P * C * 2 * 3 + P * 4, N=N,
              path="16-byte" if C % 8 == 0 else "scalar")


def run_latent(name, R, L, iters, rounds=3):
    """the Gaussian latent forward (z and kl) and backward (dstats) against torch eager mu + exp(0.5 lv) randn_like with the KL
    and its autograd, on the same bf16 stats; bytes: stats read, z written, kl written (forward); stats and dz read, dstats written
    (backward).  The kernels also run Philox, a log, a sine and cosine, a square root and two exponentials per element, so they may
    be bound by issue rather than by HBM."""
    stats, dz = _bf((R, 2 * L)), _bf((R, L), 0.1)
    z, ds, kl = torch.empty((R, L), dtype=torch.bfloat16, device="cuda"), torch.empty_like(stats), torch.empty(R, device="cuda")
    st = stats.clone().requires_grad_(True)

    def theirs():
        mu, lv = st[:, :L], st[:, L:]
        zt = mu + torch.exp(0.5 * lv) * torch.randn_like(mu)
        klt = 0.5 * (mu.float() ** 2 + torch.exp(lv.float()) - 1 - lv.float()).sum(1)
        torch.autograd.grad((zt, klt.sum() / R), st, (dz, None))
    info = pkg.gaussian_latent_info(R, L)
    best = None
    for _ in range(rounds):
        a = timed(lambda: eng.gaussian_latent_fwd(stats, z, R, L, 1, 1, kl=kl), iters)
        b = timed(lambda: eng.gaussian_latent_bwd(stats, dz, ds, R, L, 1, 1, 1.0 / R), iters)
        c = timed(theirs, iters)
        best = (a, b, c) if best is None else tuple(min(u, v) for u, v in zip(best, (a, b, c)))
    a, b, c = best
    n = R * L
    _line(f"latent {name} fwd+bwd", a + b, c, n * 16 + R * 4, R=R, L=L,
          path="16-byte" if info["vec"] == 8 else "scalar", fwd_us=a * 1e3, bwd_us=b * 1e3,
          fwd_hbm_frac=(n * 6 + R * 4) / (a * 1e-3) / 1e9 / HBM, bwd_hbm_frac=(n * 10) / (b * 1e-3) / 1e9 / HBM)


def run_bce(name, P, C, ts, iters, rounds=3):
    """the binary cross-entropy with logits (dlogits and the per-pixel loss) against F.binary_cross_entropy_with_logits forward plus
    autograd on the same bf16 tensors; bytes: logits and the C target channels read, dlogits written (bf16), the loss (fp32)"""
    x, t = _bf((P, C), 4.0), torch.rand((P, ts), device="cuda").to(torch.bfloat16)
    d, loss = torch.empty_like(x), torch.empty(P, dtype=torch.float32, device="cuda")
    xt, tt = x.clone().requires_grad_(True), t[:, :C]
    F = torch.nn.functional
    best = None
    for _ in range(rounds):
        a = timed(lambda: eng.bce_logits_loss_bf16(x, t, P, C, d, loss, target_stride=ts), iters)
        b = timed(lambda: torch.autograd.grad(F.binary_cross_entropy_with_logits(xt, tt), xt), iters)
        best = (a, b) if best is None else (min(a, best[0]), min(b, best[1]))
    _line(f"bce {name}", best[0], best[1], P * C * 2 * 3 + P * 4, P=P, C=C, target_stride=ts,
          path="16-byte" if C % 8 == 0 and ts % 8 == 0 else "scalar")


def run_vae(iters):
    """one ConvVAE training step (forward, backward, AdamW) at N = 32, and the same network in torch eager: bf16 channels-last
    convolutions (cuDNN), the latent and the loss in float32, on one fixed batch"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import vae_nets
    d = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    cls = vae_nets.ConvVAE
    B, L = cls.NB, cls.L
    p = cls.init_params()
    net = cls(eng, pkg, p)
    opt = pkg.AdamW(eng, net.layers())
    b = pkg.ImageBatcher(eng, d["train_u8"].reshape(-1, 28, 28), d["train_labels"], B, pad=2, flip=True, C_out=8)
    x = b.batch(0)[0]

    def step():
        net.forward(x)
        net.backward()
        opt.step(cls.LR)
    ms = timed(step, iters)
    F = torch.nn.functional
    cl = torch.channels_last
    w = {}
    for k, v in p.items():
        t = torch.from_numpy(v).to("cuda")
        if k in ("f1", "f2"):
            t = t.permute(0, 3, 1, 2)
        elif k in ("we", "wd", "w"):
            t = t.reshape(t.shape[0], -1)
        w[k] = t.to(torch.bfloat16).contiguous(memory_format=cl if t.dim() == 4 else torch.contiguous_format).requires_grad_(True)
    topt = torch.optim.AdamW(list(w.values()), lr=cls.LR)
    xt = torch.rand(B, 8, 28, 28, device="cuda").to(torch.bfloat16).contiguous(memory_format=cl)

    def tstep():
        h = F.relu(F.conv2d(xt, w["f1"], w["b1"], stride=2, padding=1))
        h = F.relu(F.conv2d(h, w["f2"], w["b2"], stride=2, padding=1))
        st = (h.permute(0, 2, 3, 1).reshape(B, -1) @ w["we"].t() + w["be"]).float()
        mu, lv = st[:, :L], st[:, L:]
        z = (mu + torch.exp(0.5 * lv) * torch.randn_like(mu)).to(torch.bfloat16)
        kl = 0.5 * (mu * mu + torch.exp(lv) - 1 - lv).sum(1)
        g = F.relu(z @ w["wd"].t() + w["bd"]).reshape(B, 4, 4, 16).permute(0, 3, 1, 2)
        g = F.relu(F.conv_transpose2d(g, w["t1"], w["tb1"], stride=2, padding=1))
        g = F.relu(F.conv_transpose2d(g, w["t2"], w["tb2"], stride=2, padding=1, output_padding=1))
        logits = F.pixel_shuffle(torch.einsum("nchw,oc->nohw", g, w["w"]) + w["bw"][None, :, None, None], 2)
        loss = (F.binary_cross_entropy_with_logits(logits.float(), xt[:, :1].float(), reduction="sum") + kl.sum()) / B
        topt.zero_grad(set_to_none=True)
        loss.backward()
        topt.step()
    ms_torch = timed(tstep, iters)
    gpu, power = card()
    print(json.dumps({"case": f"ConvVAE training step N={B}", "us": ms * 1e3, "torch_eager_us": ms_torch * 1e3,
                      "torch_over_ours": ms_torch / ms, "gpu": gpu, "power_limit": power}), flush=True)
    b.close()
    opt.close()
    net.close()


def run_restorer(which, iters):
    """one training step (forward, backward, AdamW) of ESPCNLite or DenoiseNet at N = 32, and the same network in torch eager: bf16
    channels-last convolutions (cuDNN) with batch norm in float32 and the loss in float32, on one fixed batch"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import restore_nets
    d = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    cls = getattr(restore_nets, which)
    p = cls.init_params()
    net = cls(eng, pkg, p)
    opt = pkg.AdamW(eng, net.layers())
    b = pkg.ImageBatcher(eng, d["train_u8"].reshape(-1, 28, 28), d["train_labels"], cls.NB, pad=2, flip=True, C_out=8)
    x = b.batch(0)[0]

    def step():
        net.forward(x)
        net.backward()
        opt.step(cls.LR)
    ms = timed(step, iters)

    F = torch.nn.functional
    cl = torch.channels_last
    w = {}
    for k, v in p.items():
        t = torch.from_numpy(v).to("cuda")
        if k.startswith("f"):
            t = t.permute(0, 3, 1, 2)
        elif k == "w":
            t = t.reshape(t.shape[0], -1)
        w[k] = t.to(torch.bfloat16).contiguous(memory_format=cl if t.dim() == 4 else torch.contiguous_format).requires_grad_(True)
    bns = [torch.nn.BatchNorm2d(c).cuda().to(memory_format=cl) for c in (16, 64)]
    bn = lambda i, v: bns[i](v.float()).to(torch.bfloat16)
    topt = torch.optim.AdamW(list(w.values()) + [q for m in bns for q in m.parameters()], lr=cls.LR)
    xt = torch.rand(cls.NB, 8, 28, 28, device="cuda").to(torch.bfloat16).contiguous(memory_format=cl)
    espcn = which == "ESPCNLite"

    def tstep():
        if espcn:
            h = F.relu(F.conv2d(F.avg_pool2d(xt, 2), w["f1"], w["b1"], padding=2))
            h = F.relu(F.conv2d(h, w["f2"], w["b2"], padding=1))
        else:
            xn = F.dropout(xt, cls.P_NOISE)
            h = F.relu(bn(0, F.conv2d(xn, w["f1"], padding=1)))
            h = F.relu(bn(1, F.conv2d(F.pixel_unshuffle(h, 2), w["f2"], padding=1)))
        out = F.pixel_shuffle(torch.einsum("nchw,oc->nohw", h, w["w"]) + w["bw"][None, :, None, None], 2)
        loss = (F.mse_loss if espcn else F.l1_loss)(out.float(), xt[:, :1].float())
        topt.zero_grad(set_to_none=True)
        loss.backward()
        topt.step()
    ms_torch = timed(tstep, iters)
    gpu, power = card()
    print(json.dumps({"case": f"{which} training step N={cls.NB}", "us": ms * 1e3, "torch_eager_us": ms_torch * 1e3,
                      "torch_over_ours": ms_torch / ms, "gpu": gpu, "power_limit": power}), flush=True)
    b.close()
    opt.close()
    net.close()


def run_dilated(name, N, H, W, C, K, R, dil, iters):
    """the three wide passes of a "same" 3x3 layer at dilation dil (padding dil), next to cuDNN (conv2d(dilation=dil) and
    aten.convolution_backward) on the same bf16 channels-last tensors and to the same layer at dilation 1 (padding 1), all in this
    run.  Bound: bytes = N * (H*W*C + P*Q*K) * 2, flops = 2 * N * P*Q*K * R*R*C, as run_wide_same."""
    pad = dil * (R - 1) // 2
    f = rng.uniform(-0.5, 0.5, (K, R, R, C)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    plans = {d: pkg.WideConvPlan(eng, N, H, W, C, K, R, R, f, b, padding=(d * (R - 1) // 2,) * 2, dilation=(d, d)) for d in {1, dil}}
    P, Q = plans[dil].out_shape[1:3]
    x = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    y = torch.empty((N, P, Q, K), dtype=torch.int16, device="cuda")
    dy = torch.randint(0, 0x3F80, (N, P, Q, K), dtype=torch.int16, device="cuda")
    dy ^= (torch.randint(0, 2, (N, P, Q, K), dtype=torch.int16, device="cuda") << 15)
    fd = torch.from_numpy(f).to("cuda")
    dw = torch.empty((K, R, R, C), dtype=torch.float32, device="cuda")
    dx = torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    xt, dyt = x.view(torch.bfloat16).permute(0, 3, 1, 2), dy.view(torch.bfloat16).permute(0, 3, 1, 2)
    wt = fd.permute(0, 3, 1, 2).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    bt = torch.from_numpy(b).to("cuda", torch.bfloat16)
    alg = N * (H * W * C + P * Q * K) * 2
    flops = 2.0 * N * P * Q * K * R * R * C
    t_bound = max(flops / 989e12, alg / 3.35e12)
    gpu, power = card()
    cb = torch.ops.aten.convolution_backward

    def passes(d):
        pd = d * (R - 1) // 2
        return (("fwd", lambda: plans[d].fwd(x, y), lambda: torch.nn.functional.conv2d(xt, wt, bt, 1, pd, d)),
                ("wgrad", lambda: eng.conv_wide_wgrad(x, dy, dw, N, H, W, C, K, R, R, padding=(pd, pd), dilation=(d, d)),
                 lambda: cb(dyt, xt, wt, None, [1, 1], [pd, pd], [d, d], False, [0, 0], 1, [False, True, False])),
                ("dgrad", lambda: eng.conv_wide_dgrad(dy, fd, dx, N, H, W, C, K, R, R, padding=(pd, pd), dilation=(d, d)),
                 lambda: cb(dyt, xt, wt, None, [1, 1], [pd, pd], [d, d], False, [0, 0], 1, [True, False, False])))

    for (what, ours, theirs), (_, ours1, theirs1) in zip(passes(dil), passes(1)):
        ms, ms_cudnn, ms1, ms1_cudnn = timed(ours, iters), timed(theirs, iters), timed(ours1, iters), timed(theirs1, iters)
        print(json.dumps({"case": f"dilated {name} d{dil} {what}", "N": N, "ms": ms, "bound_frac": t_bound / (ms * 1e-3),
                          "cudnn_ms": ms_cudnn, "cudnn_over_ours": ms_cudnn / ms, "d1_ms": ms1, "ours_over_d1": ms / ms1,
                          "cudnn_d1_ms": ms1_cudnn, "gpu": gpu, "power_limit": power}), flush=True)
    for p in plans.values():
        p.close()


def run_dwdilated(name, N, H, W, C, R, dil, iters):
    """the three passes of a "same" depthwise layer at dilation dil next to torch's conv2d(groups=C, dilation=dil) and
    aten.convolution_backward on the same bf16 channels-last tensors, and to the same layer at dilation 1 (bytes as run_dwconv)"""
    w = rng.uniform(-0.5, 0.5, (C, R, R)).astype(np.float32)
    plans = {d: pkg.DepthwiseConvPlan(eng, N, H, W, C, R, R, w, None, padding=(d * (R - 1) // 2,) * 2, dilation=(d, d)) for d in {1, dil}}
    bits = lambda *shape: torch.randint(0, 0x3F80, shape, dtype=torch.int16, device="cuda")
    x, dy = bits(N, H, W, C), bits(N, H, W, C)
    y, dx = torch.empty((N, H, W, C), dtype=torch.int16, device="cuda"), torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    dw = torch.empty((C, R, R), dtype=torch.float32, device="cuda")
    xt, dyt = x.view(torch.bfloat16).permute(0, 3, 1, 2), dy.view(torch.bfloat16).permute(0, 3, 1, 2)
    wt = torch.from_numpy(w).to("cuda").to(torch.bfloat16)[:, None].contiguous(memory_format=torch.channels_last)
    cb = torch.ops.aten.convolution_backward
    nbytes = N * 2 * H * W * C * 2
    gpu, power = card()

    def passes(d):
        pd = d * (R - 1) // 2
        return (("fwd", lambda: plans[d].fwd(x, y), lambda: torch.nn.functional.conv2d(xt, wt, None, 1, pd, d, groups=C)),
                ("dgrad", lambda: eng.dwconv_dgrad(plans[d], dy, dx),
                 lambda: cb(dyt, xt, wt, None, [1, 1], [pd, pd], [d, d], False, [0, 0], C, [True, False, False])),
                ("wgrad", lambda: eng.dwconv_wgrad(plans[d], x, dy, dw),
                 lambda: cb(dyt, xt, wt, None, [1, 1], [pd, pd], [d, d], False, [0, 0], C, [False, True, False])))

    for (what, ours, theirs), (_, ours1, _) in zip(passes(dil), passes(1)):
        ms, ms_torch, ms1 = timed(ours, iters), timed(theirs, iters), timed(ours1, iters)
        print(json.dumps({"case": f"dwdilated {name} d{dil} {what}", "N": N, "us": ms * 1e3, "share_of_3350": nbytes / (ms * 1e-3) / 1e9 / HBM,
                          "torch_us": ms_torch * 1e3, "torch_over_ours": ms_torch / ms, "d1_us": ms1 * 1e3, "ours_over_d1": ms / ms1,
                          "gpu": gpu, "power_limit": power}), flush=True)
    for p in plans.values():
        p.close()


def run_deeplab(iters):
    """one DeepLabLite training step (forward, backward, SGD with momentum) at N = 32, and the same network in torch eager: bf16
    channels-last convolutions (cuDNN) with batch norm in float32, on one fixed batch"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import deeplab_nets
    import segment_ref
    d = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    cls = deeplab_nets.DeepLabLite
    p = cls.init_params()
    net = cls(eng, pkg, p)
    opt = pkg.SGD(eng, net.layers(), momentum=0.9)
    b = pkg.ImageBatcher(eng, d["train_u8"].reshape(-1, 28, 28), d["train_labels"], cls.NB, pad=2, flip=True, C_out=8,
                         masks=segment_ref.digit_masks(d["train_u8"], d["train_labels"]))
    batch = b.batch(0)

    def step():
        net.forward(*batch)
        net.backward()
        opt.step(cls.LR)
    ms = timed(step, iters)

    F = torch.nn.functional
    cl = torch.channels_last
    w = {}
    for k, v in p.items():
        t = torch.from_numpy(v).to("cuda")
        if k == "wc":
            t = t.reshape(32, 1, 3, 3)
        elif k.startswith("f"):
            t = t.permute(0, 3, 1, 2)
        elif k == "w":
            t = t.reshape(t.shape[0], -1)
        w[k] = t.to(torch.bfloat16).contiguous(memory_format=cl if t.dim() == 4 else torch.contiguous_format).requires_grad_(True)
    bns = [torch.nn.BatchNorm2d(c).cuda().to(memory_format=cl) for c in (16, 32, 32, 32, 32, 32, 32)]
    bn = lambda i, v: bns[i](v.float()).to(torch.bfloat16)
    params = list(w.values()) + [q for m in bns for q in m.parameters()]
    topt = torch.optim.SGD(params, lr=cls.LR, momentum=0.9)
    x = torch.randn(cls.NB, 8, 28, 28, device="cuda").to(torch.bfloat16).contiguous(memory_format=cl)
    tgt = torch.randint(0, 11, (cls.NB, 28, 28), device="cuda")

    def tstep():
        a = F.relu(bn(0, F.conv2d(x, w["f1"], padding=1)))
        bb = F.relu(bn(1, F.conv2d(a, w["f2"], padding=1, stride=2)))
        m = F.relu(bn(2, F.conv2d(bb, w["fd1"], padding=2, dilation=2)))
        h = F.relu(bn(3, F.conv2d(m, w["fd2"], padding=2, dilation=2)) + bb)
        sa = bn(4, F.conv2d(m, w["fa"]))
        sb = bn(5, F.conv2d(h, w["fb"], padding=4, dilation=4)) + sa
        out = F.relu(bn(6, F.conv2d(F.conv2d(h, w["wc"], padding=6, dilation=6, groups=32), w["fp"])) + sb)
        z14 = torch.einsum("nchw,oc->nohw", out, w["w"]) + w["bw"][None, :, None, None]
        z = F.interpolate(z14, size=(28, 28), mode="bilinear", align_corners=False)
        loss = F.cross_entropy(z.float(), tgt, ignore_index=255)
        topt.zero_grad(set_to_none=True)
        loss.backward()
        topt.step()
    ms_torch = timed(tstep, iters)
    gpu, power = card()
    print(json.dumps({"case": f"DeepLabLite training step N={cls.NB}", "us": ms * 1e3, "torch_eager_us": ms_torch * 1e3,
                      "torch_over_ours": ms_torch / ms, "gpu": gpu, "power_limit": power}), flush=True)
    b.close()
    opt.close()
    net.close()


def run_wide(name, N, H, W, C, K, R, S, stride, iters):
    """the wide-channel forward (WideConvPlan) next to torch.nn.functional.conv2d (cuDNN) on the same bf16 channels-last tensors.
    Bound: the larger of flops / 989 TFLOP/s (H100 SXM dense bf16) and bytes / 3.35 TB/s, bytes = N * (H*W*C + P*Q*K) * 2."""
    P, Q = (H - R) // stride + 1, (W - S) // stride + 1
    f = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    plan = pkg.WideConvPlan(eng, N, H, W, C, K, R, S, f, b, stride=stride)
    info = pkg.conv_wide_plan_info(N, H, W, C, K, R, S, stride)
    x = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")   # positive bf16 bit patterns < 1.0
    y = torch.empty((N, P, Q, K), dtype=torch.int16, device="cuda")
    xt = x.view(torch.bfloat16).permute(0, 3, 1, 2)                                  # NCHW view of NHWC memory: channels-last
    wt = torch.from_numpy(f).permute(0, 3, 1, 2).to("cuda", torch.bfloat16).contiguous(memory_format=torch.channels_last)
    bt = torch.from_numpy(b).to("cuda", torch.bfloat16)

    def timeit(fn):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(iters):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    ms = timeit(lambda: plan.fwd(x, y))
    ms_cudnn = timeit(lambda: torch.nn.functional.conv2d(xt, wt, bt, stride=stride))
    alg = N * (H * W * C + P * Q * K) * 2
    flops = 2.0 * N * P * Q * K * R * S * C
    t_tc, t_hbm = flops / 989e12, alg / 3.35e12
    gpu, power = card()
    print(json.dumps({"case": name, "N": N, "ms": ms, "useful_TFLOPs": flops / (ms * 1e-3) / 1e12, "alg_GBps": alg / (ms * 1e-3) / 1e9,
                      "bound": "tensor" if t_tc >= t_hbm else "hbm", "bound_frac": max(t_tc, t_hbm) / (ms * 1e-3),
                      "cudnn_ms": ms_cudnn, "cudnn_bound_frac": max(t_tc, t_hbm) / (ms_cudnn * 1e-3),
                      "useful_pixel_share": info["useful_pixels"] / info["issued_pixels"], "tile": f"{info['Pt']}x{info['Qt']}",
                      "stages": info["stages"], "gpu": gpu, "power_limit": power}), flush=True)
    plan.close()
    del x, y, xt


def run_wide_bwd(name, N, H, W, C, K, R, S, stride, iters):
    """the wide-channel gradients (pcnn_conv_wide_wgrad / pcnn_conv_wide_dgrad) next to cuDNN's
    (torch.ops.aten.convolution_backward with one gradient selected) on the same bf16 channels-last tensors.  Bound as in
    run_wide: the larger of flops / 989 TFLOP/s and bytes / 3.35 TB/s, bytes = N * (H*W*C + P*Q*K) * 2 (the two tensors each
    pass reads or writes once; the filters are small)."""
    P, Q = (H - R) // stride + 1, (W - S) // stride + 1
    info = pkg.conv_wide_bwd_info(N, H, W, C, K, R, S, stride)
    x = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")   # positive bf16 bit patterns < 1.0
    dy = torch.randint(0, 0x3F80, (N, P, Q, K), dtype=torch.int16, device="cuda")
    dy ^= (torch.randint(0, 2, (N, P, Q, K), dtype=torch.int16, device="cuda") << 15)   # random signs
    f = torch.rand((K, R, S, C), dtype=torch.float32, device="cuda") - 0.5
    dw = torch.empty((K, R, S, C), dtype=torch.float32, device="cuda")
    dx = torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    xt, dyt = x.view(torch.bfloat16).permute(0, 3, 1, 2), dy.view(torch.bfloat16).permute(0, 3, 1, 2)   # channels-last views
    wt = f.permute(0, 3, 1, 2).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    alg = N * (H * W * C + P * Q * K) * 2
    flops = 2.0 * N * P * Q * K * R * S * C
    t_bound = max(flops / 989e12, alg / 3.35e12)
    gpu, power = card()

    def timeit(fn):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(iters):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    def cudnn(mask):
        return torch.ops.aten.convolution_backward(dyt, xt, wt, None, [stride, stride], [0, 0], [1, 1], False, [0, 0], 1, mask)

    for what, fn, mask in (("wgrad", lambda: eng.conv_wide_wgrad(x, dy, dw, N, H, W, C, K, R, S, stride=stride), [False, True, False]),
                           ("dgrad", lambda: eng.conv_wide_dgrad(dy, f, dx, N, H, W, C, K, R, S, stride=stride), [True, False, False])):
        ms = timeit(fn)
        ms_cudnn = timeit(lambda: cudnn(mask))
        print(json.dumps({"case": f"{name} {what}", "N": N, "ms": ms, "useful_TFLOPs": flops / (ms * 1e-3) / 1e12,
                          "bound": "tensor" if flops / 989e12 >= alg / 3.35e12 else "hbm", "bound_frac": t_bound / (ms * 1e-3),
                          "cudnn_ms": ms_cudnn, "cudnn_TFLOPs": flops / (ms_cudnn * 1e-3) / 1e12, "cudnn_bound_frac": t_bound / (ms_cudnn * 1e-3),
                          "tiling": {k: v for k, v in info.items() if k.startswith(what)}, "gpu": gpu, "power_limit": power}), flush=True)
    del x, dy, dx, xt, dyt


def run_wide_same(name, N, H, W, C, K, R, S, stride, pad, iters):
    """a "same" layer three ways, per pass: the built-in padding of the wide kernels (padding=(pad, pad)); the pad-copy route,
    each step timed alone (pcnn_pad_nhwc_bf16 into the canvas, the unpadded wide pass on the canvas, and pcnn_crop_nhwc_bf16 for
    dx); cuDNN with padding=pad on the same bf16 channels-last tensors.  Bound as in run_wide on the unpadded tensors:
    bytes = N * (H*W*C + P*Q*K) * 2, flops = 2 * N * P*Q*K * R*S*C."""
    Hc, Wc = H + 2 * pad, W + 2 * pad
    P, Q = (Hc - R) // stride + 1, (Wc - S) // stride + 1
    f = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    plan = pkg.WideConvPlan(eng, N, H, W, C, K, R, S, f, b, stride=stride, padding=(pad, pad))
    plan_c = pkg.WideConvPlan(eng, N, Hc, Wc, C, K, R, S, f, b, stride=stride)
    x = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")   # positive bf16 bit patterns < 1.0
    xc = torch.empty((N, Hc, Wc, C), dtype=torch.int16, device="cuda")
    y = torch.empty((N, P, Q, K), dtype=torch.int16, device="cuda")
    dy = torch.randint(0, 0x3F80, (N, P, Q, K), dtype=torch.int16, device="cuda")
    dy ^= (torch.randint(0, 2, (N, P, Q, K), dtype=torch.int16, device="cuda") << 15)   # random signs
    fd = torch.from_numpy(f).to("cuda")
    dw = torch.empty((K, R, S, C), dtype=torch.float32, device="cuda")
    dx = torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    dxc = torch.empty((N, Hc, Wc, C), dtype=torch.int16, device="cuda")
    xt, dyt = x.view(torch.bfloat16).permute(0, 3, 1, 2), dy.view(torch.bfloat16).permute(0, 3, 1, 2)   # channels-last views
    wt = fd.permute(0, 3, 1, 2).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    bt = torch.from_numpy(b).to("cuda", torch.bfloat16)
    alg = N * (H * W * C + P * Q * K) * 2
    flops = 2.0 * N * P * Q * K * R * S * C
    t_bound = max(flops / 989e12, alg / 3.35e12)
    gpu, power = card()

    def timeit(fn):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(iters):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    def cudnn_bwd(mask):
        return torch.ops.aten.convolution_backward(dyt, xt, wt, None, [stride, stride], [pad, pad], [1, 1], False, [0, 0], 1, mask)

    pad_ms = timeit(lambda: eng.pad_nhwc(x, xc, N, H, W, C, pad, pad))
    crop_ms = timeit(lambda: eng.crop_nhwc(dxc, dx, N, H, W, C, pad, pad))
    passes = (
        ("fwd", lambda: plan.fwd(x, y), [("pad", pad_ms), ("valid", timeit(lambda: plan_c.fwd(xc, y)))],
         lambda: torch.nn.functional.conv2d(xt, wt, bt, stride=stride, padding=pad)),
        ("wgrad", lambda: eng.conv_wide_wgrad(x, dy, dw, N, H, W, C, K, R, S, stride=stride, padding=(pad, pad)),
         [("pad", pad_ms), ("valid", timeit(lambda: eng.conv_wide_wgrad(xc, dy, dw, N, Hc, Wc, C, K, R, S, stride=stride)))],
         lambda: cudnn_bwd([False, True, False])),
        ("dgrad", lambda: eng.conv_wide_dgrad(dy, fd, dx, N, H, W, C, K, R, S, stride=stride, padding=(pad, pad)),
         [("valid", timeit(lambda: eng.conv_wide_dgrad(dy, fd, dxc, N, Hc, Wc, C, K, R, S, stride=stride))), ("crop", crop_ms)],
         lambda: cudnn_bwd([True, False, False])),
    )
    for what, fn, route, cudnn in passes:
        ms = timeit(fn)
        ms_cudnn = timeit(cudnn)
        route_ms = sum(t for _, t in route)
        print(json.dumps({"case": f"{name} {what}", "N": N, "ms": ms, "bound": "tensor" if flops / 989e12 >= alg / 3.35e12 else "hbm",
                          "bound_frac": t_bound / (ms * 1e-3), "route_ms": {k: t for k, t in route}, "route_total_ms": route_ms,
                          "route_over_builtin": route_ms / ms, "canvas_valid_over_builtin": dict(route)["valid"] / ms,
                          "cudnn_ms": ms_cudnn, "cudnn_bound_frac": t_bound / (ms_cudnn * 1e-3), "gpu": gpu, "power_limit": power}),
              flush=True)
    plan.close()
    plan_c.close()
    del x, xc, y, dy, dx, dxc, xt, dyt


def run_train(name, N, H, W, C, K, R, S, stride, pad, iters, with_dx=True, act=1):
    """one training step of a ConvLayer (bias, sigmoid at act 1, ReLU at act 3), pass by pass: forward, pcnn_conv_bias_act_bwd (out
    of place, so that every launch sees the same dy), the family's weight and input gradients, sgd (two fp32 updates and
    pcnn_conv_plan_set_params), and the whole ConvLayer step (forward, backward in place over dy, sgd).  bias_act_bwd moves
    3 * pixels * K * 2 bytes (read y and dy, write dpre), compared with 3.35 TB/s.  Next to it the torch eager step on bf16
    channels-last tensors of the same shapes: conv2d with bias, the activation, autograd backward with dy, then w -= lr * grad on
    fp32 masters and the re-cast to bf16.  At act 3 the forward of the same layer is also timed at act 0, 1 and 3, alternating
    plans of the three codes (fwd_by_act: two rounds each)."""
    Hc, Wc = H + 2 * pad, W + 2 * pad
    P, Q = (Hc - R) // stride + 1, (Wc - S) // stride + 1
    f = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    layer = pkg.ConvLayer(eng, N, H, W, C, K, R, S, f, b, act=act, stride=stride, padding=(pad, pad))
    pitch = layer.row_pitch
    x = torch.randint(0, 0x3F80, (N * H, pitch), dtype=torch.int16, device="cuda")   # positive bf16 bit patterns < 1.0
    if act == pkg.ACT_RELU:                                                           # signed x: about half the outputs < 0
        x ^= (torch.randint(0, 2, (N * H, pitch), dtype=torch.int16, device="cuda") << 15)
    y = torch.empty((N, P, Q, K), dtype=torch.int16, device="cuda")
    dy = torch.randint(0, 0x3F80, (N, P, Q, K), dtype=torch.int16, device="cuda")
    dy ^= (torch.randint(0, 2, (N, P, Q, K), dtype=torch.int16, device="cuda") << 15)   # random signs
    dpre, dy_step = torch.empty_like(dy), torch.empty_like(dy)
    dx = torch.empty_like(x) if with_dx else None
    pixels, lr = N * P * Q, 1e-6
    gpu, power = card()

    def timeit(fn):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(iters):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    args = (N, H, W, C, K, R, S)
    if layer.family == "narrow":
        wgrad = lambda: eng.conv_wgrad(x, dpre, layer.dw, *args, pitch, 0, stride)
        dgrad = lambda: eng.conv_dgrad(dpre, layer.filt, dx, *args, pitch, 0, stride)
    else:
        wgrad = lambda: eng.conv_wide_wgrad(x, dpre, layer.dw, *args, pitch, 0, stride, (pad, pad))
        dgrad = lambda: eng.conv_wide_dgrad(dpre, layer.filt, dx, *args, pitch, 0, stride, (pad, pad))

    def step():
        dy_step.copy_(dy)                          # backward consumes dy; the copy is timed on its own below
        layer.forward(x, y)
        layer.backward(y, dy_step, dx)
        layer.sgd(lr)

    ms = {"fwd": timeit(lambda: layer.forward(x, y)),
          "bias_act_bwd": timeit(lambda: eng.conv_bias_act_bwd(y, dy, dpre, layer.db, pixels, K, act)),
          "wgrad": timeit(wgrad)}
    if with_dx:
        ms["dgrad"] = timeit(dgrad)
    ms["sgd_set_params"] = timeit(lambda: layer.sgd(lr))
    ms["dy_copy"] = timeit(lambda: dy_step.copy_(dy))
    ms["layer_step_minus_dy_copy"] = timeit(step) - ms["dy_copy"]
    fwd_by_act = {}
    if act == pkg.ACT_RELU:
        layers = {a: pkg.ConvLayer(eng, N, H, W, C, K, R, S, f, b, act=a, stride=stride, padding=(pad, pad)) for a in (0, 1, 3)}
        for _ in range(2):
            for a, lay in layers.items():
                fwd_by_act.setdefault(f"act{a}", []).append(timeit(lambda: lay.forward(x, y)))
        for lay in layers.values():
            lay.close()

    # torch eager step on the same shapes (fresh random x: the values do not change the work)
    xt = x[:, :W * C].reshape(N, H, W, C).view(torch.bfloat16).permute(0, 3, 1, 2).detach().requires_grad_(with_dx)
    dyt = dy.view(torch.bfloat16).permute(0, 3, 1, 2)
    w32 = torch.from_numpy(f).permute(0, 3, 1, 2).to("cuda").contiguous(memory_format=torch.channels_last)
    b32 = torch.from_numpy(b).to("cuda")
    wb, bb = w32.to(torch.bfloat16).requires_grad_(True), b32.to(torch.bfloat16).requires_grad_(True)

    def torch_step():
        wb.grad = bb.grad = None
        if with_dx:
            xt.grad = None
        out = torch.nn.functional.conv2d(xt, wb, bb, stride=stride, padding=pad)
        out = torch.relu(out) if act == pkg.ACT_RELU else torch.sigmoid(out)
        out.backward(dyt)
        with torch.no_grad():
            w32.add_(wb.grad.float(), alpha=-lr)
            b32.add_(bb.grad.float(), alpha=-lr)
            wb.copy_(w32)
            bb.copy_(b32)

    ms["torch_eager_step"] = timeit(torch_step)
    ba_bytes = 3 * pixels * K * 2
    print(json.dumps({"case": name, "act": act, "N": N, "family": layer.family, "dx": with_dx, "ms": ms, "fwd_by_act_ms": fwd_by_act,
                      "bias_act_GBps": ba_bytes / (ms["bias_act_bwd"] * 1e-3) / 1e9,
                      "bias_act_hbm_frac": ba_bytes / (ms["bias_act_bwd"] * 1e-3) / 1e9 / HBM,
                      "layer_over_torch": ms["layer_step_minus_dy_copy"] / ms["torch_eager_step"], "gpu": gpu, "power_limit": power}),
          flush=True)
    layer.close()
    del x, y, dy, dpre, dy_step, dx, xt


def run_pool(name, N, H, W, C, R, stride, pad, iters):
    """the NHWC max pool (pcnn_maxpool_nhwc_bf16_fwd / _bwd) next to torch's max_pool2d(return_indices=True) and
    max_pool2d_with_indices_backward on the same channels-last bf16 tensors.  Bytes: forward N*H*W*C*2 + N*P*Q*C*3 (read x, write
    y and the one-byte argmax), backward N*P*Q*C*3 + N*H*W*C*2 (read dy and argmax, write dx); re-reads of x by overlapping
    windows come from L2 and are not counted.  Torch's forward writes 8-byte indices: N*P*Q*C*10 bytes on its output side."""
    P, Q = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1
    x = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")   # positive bf16 bit patterns < 1.0
    x ^= (torch.randint(0, 2, (N, H, W, C), dtype=torch.int16, device="cuda") << 15)   # random signs
    y = torch.empty((N, P, Q, C), dtype=torch.int16, device="cuda")
    am = torch.empty((N, P, Q, C), dtype=torch.uint8, device="cuda")
    dy = torch.randint(0, 0x3F80, (N, P, Q, C), dtype=torch.int16, device="cuda")
    dy ^= (torch.randint(0, 2, (N, P, Q, C), dtype=torch.int16, device="cuda") << 15)
    dx = torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    xt, dyt = x.view(torch.bfloat16).permute(0, 3, 1, 2), dy.view(torch.bfloat16).permute(0, 3, 1, 2)   # channels-last views
    _, idx = torch.nn.functional.max_pool2d(xt, R, stride, pad, return_indices=True)
    gpu, power = card()

    def timeit(fn):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(iters):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    big, small = N * H * W * C, N * P * Q * C
    args = (N, H, W, C, R, R, stride, (pad, pad))
    eng.maxpool_nhwc_fwd(x, y, am, *args)                          # the backward reads this argmax
    for what, fn, tfn, nbytes in (
            ("fwd", lambda: eng.maxpool_nhwc_fwd(x, y, am, *args),
             lambda: torch.nn.functional.max_pool2d(xt, R, stride, pad, return_indices=True), big * 2 + small * 3),
            ("bwd", lambda: eng.maxpool_nhwc_bwd(dy, am, dx, *args),
             lambda: torch.ops.aten.max_pool2d_with_indices_backward(dyt, xt, [R, R], [stride, stride], [pad, pad], [1, 1], False, idx),
             small * 3 + big * 2)):
        ms, ms_torch = timeit(fn), timeit(tfn)
        print(json.dumps({"case": f"{name} {what}", "N": N, "ms": ms, "GBps": nbytes / (ms * 1e-3) / 1e9,
                          "hbm_frac": nbytes / (ms * 1e-3) / 1e9 / HBM, "torch_ms": ms_torch, "torch_over_ours": ms_torch / ms,
                          "vec": pkg.maxpool_nhwc_info(*args[:7], args[7])["vec"], "gpu": gpu, "power_limit": power}), flush=True)
    del x, y, am, dy, dx, xt, dyt, idx


def run_nlblock(name, N, H, W, C, h, d, iters):
    """one non-local block training step (forward and backward, no optimizer): SelfAttentionLayer then BatchNormLayer with r = the
    block's input, against the same block in torch eager (bf16 linear layers, scaled_dot_product_attention, batch norm and the
    residual, autograd for the input and parameter gradients)"""
    hd, T = h * d, H * W
    g = np.random.default_rng(5)
    wq, bq = (g.standard_normal((3 * hd, C)) / np.sqrt(C)).astype(np.float32), np.zeros(3 * hd, np.float32)
    wo, bo = (g.standard_normal((C, hd)) / np.sqrt(hd)).astype(np.float32), np.zeros(C, np.float32)
    attn = pkg.SelfAttentionLayer(eng, N, H, W, C, h, d, wq, bq, wo, bo)
    bn = pkg.BatchNormLayer(eng, N, H, W, C)
    x, dz = _bf((N, H, W, C)), _bf((N, H, W, C))
    wz, z, dwz, dres, dx = (torch.empty_like(x) for _ in range(5))

    def step():
        attn.forward(x, wz)
        bn.forward(wz, z, r=x)
        bn.backward(z, dz, dwz, dr=dres)
        attn.backward(dwz, dx)

    ms = timed(step, iters)
    tq, tbq, to, tbo = (torch.tensor(a, device="cuda", dtype=torch.bfloat16, requires_grad=True) for a in (wq, bq, wo, bo))
    gamma, beta = (torch.full((C,), v, device="cuda", requires_grad=True) for v in (1.0, 0.0))
    xt = x.detach().clone().requires_grad_(True)

    def torch_step():
        t = xt.reshape(N, T, C)
        q, k, v = torch.nn.functional.linear(t, tq, tbq).reshape(N, T, 3, h, d).permute(2, 0, 3, 1, 4)
        o = torch.nn.functional.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(N, T, hd)
        y = torch.nn.functional.linear(o, to, tbo).reshape(N, H, W, C).permute(0, 3, 1, 2)
        zt = torch.nn.functional.batch_norm(y, None, None, gamma, beta, training=True) + xt.permute(0, 3, 1, 2)
        torch.autograd.grad(zt, (xt, tq, tbq, to, tbo, gamma, beta), dz.permute(0, 3, 1, 2))

    ms_t = timed(torch_step, iters)
    _line(name, ms, ms_t)
    attn.close()
    bn.close()


def run_attn(name, N, T, h, d, iters):
    """self-attention forward and backward (pcnn_attention_bf16_fwd / _bwd) against torch's flash scaled_dot_product_attention
    and its autograd backward, on the same bf16 [N][T][h][d] tensors.  Useful work: 4 N h T^2 d flops forward, 10 N h T^2 d
    backward (the five T x T x d products, without the recomputed S); the backward recomputes S, a further 2 N h T^2 d, reported
    apart.  Shares of the 989 TFLOP/s dense bf16 data-sheet figure."""
    q, k, v, do = (_bf((N, T, h, d)) for _ in range(4))
    o = torch.empty_like(q)
    lse = torch.empty((N, h, T), device="cuda", dtype=torch.float32)
    dq, dk, dv = (torch.empty_like(q) for _ in range(3))
    fwd = lambda: eng.attention_fwd(q, k, v, o, lse, N, T, h, d)
    bwd = lambda: eng.attention_bwd(q, k, v, o, do, lse, dq, dk, dv, N, T, h, d)
    fwd()
    ms_f, ms_b = timed(fwd, iters), timed(bwd, iters)
    from torch.nn.attention import SDPBackend, sdpa_kernel
    qt, kt, vt = (t.transpose(1, 2).detach().requires_grad_(True) for t in (q, k, v))
    dot = do.transpose(1, 2)
    with sdpa_kernel(SDPBackend.FLASH_ATTENTION):
        ot = torch.nn.functional.scaled_dot_product_attention(qt, kt, vt)
        ms_tf = timed(lambda: torch.nn.functional.scaled_dot_product_attention(qt, kt, vt), iters)
        ms_tb = timed(lambda: torch.autograd.grad(ot, (qt, kt, vt), dot, retain_graph=True), iters)
    diff = (o.float() - ot.detach().transpose(1, 2).float()).abs().max().item()
    fl = N * h * T * T * d
    peak = 989e12
    _line(name + " fwd", ms_f, ms_tf, flops=4 * fl, tflops=4 * fl / ms_f / 1e9, peak_frac=4 * fl / (ms_f * 1e-3) / peak, max_abs_diff_o=diff)
    _line(name + " bwd", ms_b, ms_tb, flops=10 * fl, recompute_flops=2 * fl, tflops=10 * fl / ms_b / 1e9,
          peak_frac=10 * fl / (ms_b * 1e-3) / peak, peak_frac_with_recompute=12 * fl / (ms_b * 1e-3) / peak)


def timed(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(iters):
        fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def run_linear(name, N, P, Q, C, O, act, iters):
    """the three passes of a LinearPlan (pcnn_conv_tc_fwd on a linear plan, pcnn_linear_wgrad, pcnn_linear_dgrad) next to
    torch.nn.functional.linear and its two backward matmuls on the same bf16 tensors.  Bound: the larger of 2 N F O / 989 TFLOP/s
    and the bytes of each operand crossing HBM once / 3.35 TB/s.  Forward: x, W bf16, y; weight gradient: x, dy, dW fp32; input
    gradient: dy, W, dx.  The fp32 slots of a split reduction (written and read once each) are reported apart: the bound omits them."""
    F_ = P * Q * C
    w = rng.uniform(-1, 1, (O, P, Q, C)).astype(np.float32) / np.float32(np.sqrt(F_))
    b = rng.uniform(-0.5, 0.5, O).astype(np.float32)
    plan = pkg.LinearPlan(eng, N, P, Q, C, O, w, b, act=act)
    info = pkg.linear_info(N, P, Q, C, O)
    pitch = info["row_pitch"]
    x = torch.randint(0, 0x3F80, (N, P, pitch), dtype=torch.int16, device="cuda")
    y = torch.empty((N, O), dtype=torch.int16, device="cuda")
    dy = torch.randint(0, 0x3F80, (N, O), dtype=torch.int16, device="cuda")
    dx = torch.empty_like(x)
    dw = eng.array((O, P, Q, C))
    gpu, power = card()
    xt = x.view(torch.bfloat16)[:, :, :Q * C].reshape(N, F_)
    wt = torch.from_numpy(w).reshape(O, F_).to("cuda").to(torch.bfloat16)
    bt = torch.from_numpy(b).to("cuda").to(torch.bfloat16)
    dyt = dy.view(torch.bfloat16)
    flops = 2.0 * N * F_ * O
    passes = (("fwd", lambda: plan.fwd(x, y), lambda: torch.nn.functional.linear(xt, wt, bt), N * F_ * 2 + O * F_ * 2 + N * O * 2,
               info["fwd_splits"], 2 * info["fwd_splits"] * N * O * 4 if info["fwd_splits"] > 1 else 0),
              ("wgrad", lambda: eng.linear_wgrad(plan, x, dy, dw), lambda: dyt.t() @ xt, N * F_ * 2 + N * O * 2 + O * F_ * 4,
               info["wgrad_splits"], 2 * info["wgrad_splits"] * O * F_ * 4 if info["wgrad_splits"] > 1 else 0),
              ("dgrad", lambda: eng.linear_dgrad(plan, dy, dx), lambda: dyt @ wt, N * O * 2 + O * F_ * 2 + N * F_ * 2, 1, 0))
    for what, fn, tfn, nbytes, splits, slot_bytes in passes:
        ms, ms_torch = timed(fn, iters), timed(tfn, iters)
        t_bound = max(flops / 989e12, nbytes / (HBM * 1e9))
        print(json.dumps({"case": f"{name} {what}", "N": N, "F": F_, "O": O, "us": ms * 1e3, "bound_us": t_bound * 1e6,
                          "bound_frac": t_bound / (ms * 1e-3), "bound_by": "flops" if flops / 989e12 > nbytes / (HBM * 1e9) else "HBM",
                          "MB": nbytes / 1e6, "splits": splits, "slot_MB": slot_bytes / 1e6, "torch_us": ms_torch * 1e3,
                          "torch_over_ours": ms_torch / ms, "gpu": gpu, "power_limit": power}), flush=True)
    plan.close()
    dw.free()
    del x, y, dy, dx


def run_classifier(N, iters, relu=False):
    """one training step of conv 8@5x5 sigmoid -> pool 2 -> conv 16@3x3 pad 1 -> pool 2 -> fc 576->128 sigmoid -> fc 128->10 ->
    softmax cross-entropy (pcnn_softmax_ce_bf16, scale 1/N) -> backward -> sgd of all four layers, on the engine's stream; next to it
    the torch eager step of the same layers on bf16 channels-last tensors (fp32 masters, w -= lr * grad, re-cast to bf16).
    relu=True: ReLU after conv 1, conv 2 and fc 1 (step 0.05)."""
    r = np.random.default_rng(5)
    u = lambda shape, fan: r.uniform(-1, 1, shape).astype(np.float32) / np.float32(np.sqrt(fan))
    p = dict(f1=u((8, 5, 5, 1), 25), b1=u(8, 25), f2=u((16, 3, 3, 8), 72), b2=u(16, 72), w3=u((128, 6, 6, 16), 576),
             b3=u(128, 576), w4=u((10, 1, 1, 128), 128), b4=u(10, 128))
    a1, a2 = (pkg.ACT_RELU, pkg.ACT_RELU) if relu else (pkg.ACT_SIGMOID, pkg.ACT_NONE)
    c1 = pkg.ConvLayer(eng, N, 28, 28, 1, 8, 5, 5, p["f1"], p["b1"], act=a1)
    c2 = pkg.ConvLayer(eng, N, 12, 12, 8, 16, 3, 3, p["f2"], p["b2"], act=a2, padding=(1, 1))
    fc1 = pkg.LinearLayer(eng, N, 6, 6, 16, 128, p["w3"], p["b3"], act=a1)
    fc2 = pkg.LinearLayer(eng, N, 1, 1, 128, 10, p["w4"], p["b4"], act=0, row_pitch=128)
    p1 = pkg.MaxPoolLayer(eng, N, 24, 24, 8, 2, row_pitch=c2.row_pitch, image_rows=c2.image_rows)
    p2 = pkg.MaxPoolLayer(eng, N, 12, 12, 16, 2, row_pitch=fc1.row_pitch, image_rows=fc1.image_rows)
    e = lambda *s: torch.empty(s, dtype=torch.int16, device="cuda")
    x = torch.randint(0, 0x3F80, (N * 28, 32), dtype=torch.int16, device="cuda")
    labels = torch.randint(0, 10, (N,), dtype=torch.uint8, device="cuda")
    y1, dy1, x2, dx2, y2, dy2 = e(N, 24, 24, 8), e(N, 24, 24, 8), e(N, 12, 96), e(N, 12, 96), e(N, 12, 12, 16), e(N, 12, 12, 16)
    x3, dx3, y3, dy3, z, dz = e(N, 6, 96), e(N, 6, 96), e(N, 128), e(N, 128), e(N, 10), e(N, 10)
    loss = torch.empty(N, dtype=torch.float32, device="cuda")
    lr = 0.05 if relu else 0.3
    gpu, power = card()

    def step():
        c1.forward(x, y1); p1.forward(y1, x2); c2.forward(x2, y2); p2.forward(y2, x3); fc1.forward(x3, y3); fc2.forward(y3, z)
        eng.softmax_ce_bf16(z, labels, N, 10, 1.0 / N, dz, loss)
        fc2.backward(z, dz, dy3); fc1.backward(y3, dy3, dx3); p2.backward(dx3, dy2); c2.backward(y2, dy2, dx2)
        p1.backward(dx2, dy1); c1.backward(y1, dy1, None)
        for layer in (c1, c2, fc1, fc2):
            layer.sgd(lr)

    ms = timed(step, iters)
    F = torch.nn.functional
    xt = x[:, :28].reshape(N, 28, 28, 1).view(torch.bfloat16).permute(0, 3, 1, 2)
    lt = labels.long()
    m32 = {k: torch.from_numpy(v).to("cuda") for k, v in p.items()}
    m32["f1"] = m32["f1"].permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
    m32["f2"] = m32["f2"].permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
    m32["w3"], m32["w4"] = m32["w3"].reshape(128, -1), m32["w4"].reshape(10, -1)
    mb = {k: v.to(torch.bfloat16).requires_grad_(True) for k, v in m32.items()}

    def torch_step():
        for v in mb.values():
            v.grad = None
        act1, act2 = (torch.relu, torch.relu) if relu else (torch.sigmoid, lambda t: t)
        h = F.max_pool2d(act1(F.conv2d(xt, mb["f1"], mb["b1"])), 2)
        h = F.max_pool2d(act2(F.conv2d(h, mb["f2"], mb["b2"], padding=1)), 2)
        h = act1(F.linear(h.permute(0, 2, 3, 1).reshape(N, -1), mb["w3"], mb["b3"]))
        F.cross_entropy(F.linear(h, mb["w4"], mb["b4"]), lt).backward()
        with torch.no_grad():
            for k in m32:
                m32[k].add_(mb[k].grad.float(), alpha=-lr)
                mb[k].copy_(m32[k])

    ms_torch = timed(torch_step, iters)
    print(json.dumps({"case": f"classifier training step N={N}" + (" ReLU" if relu else ""), "ms": ms, "torch_eager_ms": ms_torch, "ours_over_torch": ms / ms_torch,
                      "gpu": gpu, "power_limit": power}), flush=True)
    for layer in (c1, c2, fc1, fc2, p1, p2):
        layer.close()


def run_bn(name, N, H, W, C, iters):
    """batch normalization with ReLU (pcnn_batchnorm_nhwc_bf16_fwd / _bwd), each pass with and without the residual r, next to
    torch's F.batch_norm (+ add) + relu and its autograd backward on the same channels-last bf16 tensors.  Bytes, T = N*H*W*C*2:
    training forward 3T (x read twice: once for the statistics, once for y; y written), eval forward 2T, + T for reading r;
    backward 7T (x, y, dy read by the statistics pass; x, y, dy read and dx written by the second), + T for writing dr.  The
    per-CTA slots (a few 100 kB) and the [C] vectors are not counted."""
    M = N * H * W
    T = M * C * 2
    rnd = lambda: torch.randint(-0x4000, 0x4000, (M, C), dtype=torch.int16, device="cuda") & 0x3FFF | 0x3C00   # bf16 in [1, 2) * 2^k
    x, r, dy = rnd(), rnd(), rnd()
    r ^= torch.randint(0, 2, (M, C), dtype=torch.int16, device="cuda") << 15
    dy ^= torch.randint(0, 2, (M, C), dtype=torch.int16, device="cuda") << 15
    y, dx, dr = (torch.empty((M, C), dtype=torch.int16, device="cuda") for _ in range(3))
    info = pkg.batchnorm_nhwc_info(M, C)
    f = lambda v: eng.to_device(np.full(C, v, np.float32))
    gamma, beta, rm, rv, sm, sr, dg, db = f(1), f(0), f(0), f(1), f(0), f(1), f(0), f(0)
    gpu, power = card()
    F = torch.nn.functional
    bf = lambda t: t.view(torch.bfloat16).reshape(N, H, W, C).permute(0, 3, 1, 2)         # channels-last NCHW views
    xt, rt, dyt = bf(x).detach().clone().requires_grad_(True), bf(r).detach().clone().requires_grad_(True), bf(dy)
    gt, bt = torch.ones(C, device="cuda", requires_grad=True), torch.zeros(C, device="cuda", requires_grad=True)
    rmt, rvt = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")

    def torch_fwd(with_r, training):
        v = F.batch_norm(xt, rmt, rvt, gt, bt, training=training, momentum=0.1, eps=1e-5)
        return torch.relu(v + rt if with_r else v)

    eng.batchnorm_fwd(x, y, M, C, gamma, beta, rm, rv, sm, sr, act=3)       # the statistics the backward reads
    for with_r in (False, True):
        rr, drr = (r, dr) if with_r else (None, None)
        out = torch_fwd(with_r, True)
        ins = [xt, gt, bt] + ([rt] if with_r else [])
        passes = (("training fwd", lambda: eng.batchnorm_fwd(x, y, M, C, gamma, beta, rm, rv, sm, sr, r=rr, act=3),
                   lambda: torch_fwd(with_r, True), 3 * T + (T if with_r else 0)),
                  ("eval fwd", lambda: eng.batchnorm_fwd(x, y, M, C, gamma, beta, rm, rv, r=rr, act=3, training=False),
                   lambda: torch_fwd(with_r, False), 2 * T + (T if with_r else 0)),
                  ("bwd", lambda: eng.batchnorm_bwd(x, y, dy, gamma, sm, sr, dx, dg, db, M, C, act=3, dr=drr),
                   lambda: torch.autograd.grad(out, ins, dyt, retain_graph=True), 7 * T + (T if with_r else 0)))
        for what, fn, tfn, nbytes in passes:
            ms, ms_torch = timed(fn, iters), timed(tfn, iters)
            print(json.dumps({"case": f"{name} {what}" + (" + r" if with_r else ""), "N": N, "us": ms * 1e3, "MB": nbytes / 1e6,
                              "hbm_frac": nbytes / (ms * 1e-3) / 1e9 / HBM, "torch_us": ms_torch * 1e3, "torch_over_ours": ms_torch / ms,
                              "vec": info["vec"], "slots": info["grad_slots"], "gpu": gpu, "power_limit": power}), flush=True)
    for a in (gamma, beta, rm, rv, sm, sr, dg, db):
        a.free()
    del x, r, dy, y, dx, dr, xt, rt


def run_resblock(N, iters):
    """one training step of a ResNet basic block, 56x56x64 at N = 128: conv_a 3x3 pad 1 (no bias) -> BN + ReLU -> conv_b -> BN + x0
    -> ReLU, its backward (dx0 and the shortcut's gradient dres left apart: the BN that wrote x0 adds them as dy2) and the sgd of
    the four layers, on the engine's stream.  Next to it the torch eager step of the same block on bf16 channels-last tensors (fp32
    masters, w -= lr * grad, re-cast to bf16)."""
    H = W = 56
    C = 64
    r = np.random.default_rng(11)
    u = lambda shape, fan: r.uniform(-1, 1, shape).astype(np.float32) / np.float32(np.sqrt(fan))
    fa, fb = u((C, 3, 3, C), 9 * C), u((C, 3, 3, C), 9 * C)
    ca = pkg.ConvLayer(eng, N, H, W, C, C, 3, 3, fa, None, act=0, padding=(1, 1))
    cb = pkg.ConvLayer(eng, N, H, W, C, C, 3, 3, fb, None, act=0, padding=(1, 1))
    ba, bb = pkg.BatchNormLayer(eng, N, H, W, C, act=pkg.ACT_RELU), pkg.BatchNormLayer(eng, N, H, W, C, act=pkg.ACT_RELU)
    e = lambda: torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    x0 = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    dout = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    dout ^= torch.randint(0, 2, (N, H, W, C), dtype=torch.int16, device="cuda") << 15
    ya, za, yb, out, dyb, dres, dza, dya, dx0 = (e() for _ in range(9))
    lr = 0.05
    gpu, power = card()

    def step():
        ca.forward(x0, ya); ba.forward(ya, za); cb.forward(za, yb); bb.forward(yb, out, r=x0)
        bb.backward(out, dout, dyb, dr=dres); cb.backward(yb, dyb, dza); ba.backward(za, dza, dya); ca.backward(ya, dya, dx0)
        for layer in (ca, ba, cb, bb):
            layer.sgd(lr)

    ms = timed(step, iters)
    F = torch.nn.functional
    xt = x0.view(torch.bfloat16).permute(0, 3, 1, 2).detach().requires_grad_(True)
    dt = dout.view(torch.bfloat16).permute(0, 3, 1, 2)
    m32 = {k: torch.from_numpy(v).to("cuda").permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last) for k, v in
           (("fa", fa), ("fb", fb))}
    m32.update(ga=torch.ones(C, device="cuda"), ba=torch.zeros(C, device="cuda"), gb=torch.ones(C, device="cuda"), bb=torch.zeros(C, device="cuda"))
    mb = {k: (v.to(torch.bfloat16) if k.startswith("f") else v.clone()).requires_grad_(True) for k, v in m32.items()}
    stats = [torch.zeros(C, device="cuda"), torch.ones(C, device="cuda"), torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")]

    def torch_step():
        for v in mb.values():
            v.grad = None
        xt.grad = None
        h = torch.relu(F.batch_norm(F.conv2d(xt, mb["fa"], padding=1), stats[0], stats[1], mb["ga"], mb["ba"], training=True))
        h = torch.relu(F.batch_norm(F.conv2d(h, mb["fb"], padding=1), stats[2], stats[3], mb["gb"], mb["bb"], training=True) + xt)
        h.backward(dt)
        with torch.no_grad():
            for k in m32:
                m32[k].add_(mb[k].grad.float(), alpha=-lr)
                mb[k].copy_(m32[k])

    ms_torch = timed(torch_step, iters)
    print(json.dumps({"case": f"basic block 56x56x64 training step N={N}", "ms": ms, "torch_eager_ms": ms_torch, "ours_over_torch": ms / ms_torch,
                      "gpu": gpu, "power_limit": power}), flush=True)
    for layer in (ca, cb, ba, bb):
        layer.close()


def run_avgpool(name, N, H, W, C, R, stride, pad, cip, iters):
    """the NHWC average pool (pcnn_avgpool_nhwc_bf16_fwd / _bwd) next to torch's avg_pool2d and avg_pool2d_backward on the same
    channels-last bf16 tensors.  Bytes: forward N*H*W*C*2 + N*P*Q*C*2 (read x, write y), backward the same (read dy, write dx);
    re-reads of x or dy by overlapping windows come from L2 and are not counted."""
    P, Q = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1
    x = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    x ^= (torch.randint(0, 2, (N, H, W, C), dtype=torch.int16, device="cuda") << 15)
    y = torch.empty((N, P, Q, C), dtype=torch.int16, device="cuda")
    dy = torch.randint(0, 0x3F80, (N, P, Q, C), dtype=torch.int16, device="cuda")
    dx = torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    xt, dyt = x.view(torch.bfloat16).permute(0, 3, 1, 2), dy.view(torch.bfloat16).permute(0, 3, 1, 2)   # channels-last views
    gpu, power = card()
    nbytes = (N * H * W * C + N * P * Q * C) * 2
    args = (N, H, W, C, R, R, stride, (pad, pad), cip)
    for what, fn, tfn in (
            ("fwd", lambda: eng.avgpool_nhwc_fwd(x, y, *args),
             lambda: torch.nn.functional.avg_pool2d(xt, R, stride, pad, count_include_pad=bool(cip))),
            ("bwd", lambda: eng.avgpool_nhwc_bwd(dy, dx, *args),
             lambda: torch.ops.aten.avg_pool2d_backward(dyt, xt, [R, R], [stride, stride], [pad, pad], False, bool(cip), None))):
        ms, ms_torch = timed(fn, iters), timed(tfn, iters)
        print(json.dumps({"case": f"{name} {what}", "N": N, "us": ms * 1e3, "MB": nbytes / 1e6, "hbm_frac": nbytes / (ms * 1e-3) / 1e9 / HBM,
                          "torch_us": ms_torch * 1e3, "torch_over_ours": ms_torch / ms,
                          "vec": pkg.avgpool_nhwc_info(*args[:7], args[7])["vec"], "gpu": gpu, "power_limit": power}), flush=True)
    del x, y, dy, dx, xt, dyt


def run_gap(name, N, H, W, C, iters):
    """global average pooling (pcnn_global_avgpool_nhwc_bf16_fwd / _bwd) next to torch's x.mean((2, 3)), adaptive_avg_pool2d(x, 1)
    and the autograd backward of the mean on the same channels-last bf16 tensors.  Bytes: forward N*H*W*C*2 + N*C*2 (read x, write
    y), backward the same (read dy, write dx).  The forward's fp32 slots (written and read once, when an image has several pixel
    ranges) are reported apart as slot_MB."""
    info = pkg.global_avgpool_nhwc_info(N, H, W, C)
    x = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    y = torch.empty((N, info["row_pitch"]), dtype=torch.int16, device="cuda")
    dy = torch.randint(0, 0x3F80, (N, info["row_pitch"]), dtype=torch.int16, device="cuda")
    dx = torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    xt = x.view(torch.bfloat16).permute(0, 3, 1, 2)
    xg = xt.detach().clone().requires_grad_(True)
    mean = xg.mean((2, 3))
    dyt = dy.view(torch.bfloat16)[:, :C]
    gpu, power = card()
    nbytes = (N * H * W * C + N * C) * 2
    slot_bytes = 2 * N * info["ranges"] * C * 4 if info["ranges"] > 1 else 0
    for what, fn, tfn, tname in (
            ("fwd", lambda: eng.global_avgpool_nhwc_fwd(x, y, N, H, W, C), lambda: xt.mean((2, 3)), "mean"),
            ("fwd", lambda: eng.global_avgpool_nhwc_fwd(x, y, N, H, W, C), lambda: torch.nn.functional.adaptive_avg_pool2d(xt, 1),
             "adaptive_avg_pool2d"),
            ("bwd", lambda: eng.global_avgpool_nhwc_bwd(dy, dx, N, H, W, C), lambda: torch.autograd.grad(mean, xg, dyt, retain_graph=True),
             "mean autograd")):
        ms, ms_torch = timed(fn, iters), timed(tfn, iters)
        print(json.dumps({"case": f"{name} {what}", "N": N, "us": ms * 1e3, "MB": nbytes / 1e6, "hbm_frac": nbytes / (ms * 1e-3) / 1e9 / HBM,
                          "slot_MB": slot_bytes / 1e6 if what == "fwd" else 0, "ranges": info["ranges"], "ctas": info["ctas"],
                          "torch": tname, "torch_us": ms_torch * 1e3, "torch_over_ours": ms_torch / ms, "vec": info["vec"], "gpu": gpu,
                          "power_limit": power}), flush=True)
    del x, y, dy, dx, xt, xg, mean


def run_resnetgap(N, iters):
    """one training step of the GAP ResNet of tests/example_nets.py (test_resnet_gap_mnist) at batch N: forward, softmax
    cross-entropy, backward and the sgd of every layer on the engine's stream; next to it the torch eager step of the same layers on
    bf16 channels-last tensors (fp32 masters, w -= lr * grad, re-cast to bf16)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from example_nets import ResNetGAP
    assert N == ResNetGAP.NB
    p = ResNetGAP.init_params()
    net = ResNetGAP(eng, pkg, p)
    xl = torch.randint(0, 0x3F80, (N * 28, 32), dtype=torch.int16, device="cuda")
    labels = torch.randint(0, 10, (N,), dtype=torch.uint8, device="cuda")
    lr = ResNetGAP.LR_STEP
    gpu, power = card()

    def step():
        net.forward(xl.data_ptr(), labels)
        net.backward()
        net.sgd(lr)

    ms = timed(step, iters)
    net.close()
    F = torch.nn.functional
    xt = xl[:, :28].reshape(N, 28, 28, 1).view(torch.bfloat16).permute(0, 3, 1, 2)
    lt = labels.long()
    m32 = {k: torch.from_numpy(v).to("cuda") for k, v in p.items()}
    for k in [k for k in m32 if k.startswith("f")]:
        m32[k] = m32[k].permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
    m32["w8"] = m32["w8"].reshape(10, -1)
    for i, c in enumerate((8, 16, 16, 16, 32, 32, 32)):
        m32[f"g{i}"], m32[f"b{i}"] = torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
    mb = {k: (v.to(torch.bfloat16) if k[0] == "f" or k in ("w8", "b8") else v.clone()).requires_grad_(True) for k, v in m32.items()}
    stats = [(torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")) for c in (8, 16, 16, 16, 32, 32, 32)]
    bn = lambda i, v: F.batch_norm(v, *stats[i], mb[f"g{i}"], mb[f"b{i}"], training=True)

    def torch_step():
        for v in mb.values():
            v.grad = None
        h = F.avg_pool2d(F.relu(bn(0, F.conv2d(xt, mb["f1"]))), 2)
        x0 = F.relu(bn(1, F.conv2d(h, mb["f2"], padding=1)))
        h = F.relu(bn(2, F.conv2d(x0, mb["f3"], padding=1)))
        x1 = F.relu(bn(3, F.conv2d(h, mb["f4"], padding=1)) + x0)
        h = F.relu(bn(4, F.conv2d(x1, mb["f5"], padding=1, stride=2)))
        s = bn(6, F.conv2d(x1, mb["f7"], padding=1, stride=2))
        h = F.relu(bn(5, F.conv2d(h, mb["f6"], padding=1)) + s)
        F.cross_entropy(F.linear(F.adaptive_avg_pool2d(h, 1).flatten(1).to(torch.bfloat16), mb["w8"], mb["b8"]), lt).backward()
        with torch.no_grad():
            for k in m32:
                m32[k].add_(mb[k].grad.float(), alpha=-lr)
                mb[k].copy_(m32[k])

    ms_torch = timed(torch_step, iters)
    print(json.dumps({"case": f"GAP ResNet training step N={N}", "ms": ms, "torch_eager_ms": ms_torch, "ours_over_torch": ms / ms_torch,
                      "gpu": gpu, "power_limit": power}), flush=True)


def run_optim(iters):
    """one fused optimizer step (pcnn_optim_step) over the 62 tensors of ResNet-18 (tests/optim_ref.py, 11.69 M fp32 elements) with
    the 19 convolutions of C % 8 == 0 carrying wide plans created at N = 1 with their real spatial sizes (a 512-filter convolution is
    two 256-filter plans over the two halves of its KRSC master: the wide plan takes K <= 256), whose bf16 operands the step rewrites;
    conv1 (C = 3) and the fc carry none.  Bytes per element: SGD with momentum reads p, g, b and writes p, b (20), AdamW reads p, g, m,
    v and writes p, m, v (28), plus 2 per operand element.  Beside it torch's fused SGD / AdamW on the same fp32 tensors, and
    torch._foreach_copy_ of the 19 masters into bf16 copies (the operand refresh torch would need)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import optim_ref as OR
    gpu, power = card()
    gen = torch.Generator(device="cuda").manual_seed(5)
    ps, gs, table, plans, op_src, n_op = [], [], [], [], [], 0
    for name, shape, h in OR.resnet18_tensors():
        n = int(np.prod(shape))
        p = torch.randn(n, device="cuda", generator=gen) * 0.05
        g = torch.randn(n, device="cuda", generator=gen) * 1e-2
        ps.append(p)
        gs.append(g)
        if len(shape) == 4 and h > 0 and shape[3] % 8 == 0:
            K, R_, S, C = shape
            stride = 2 if (".0.conv1" in name or ".0.down" in name) and not name.startswith("layer1") else 1
            host_f = p.cpu().numpy().reshape(shape)
            for k0 in range(0, K, 256):
                k = min(256, K - k0)
                plan = pkg.WideConvPlan(eng, 1, h, h, C, k, R_, S, host_f[k0:k0 + k], None, stride=stride, padding=(R_ // 2, S // 2))
                plans.append(plan)
                off = k0 * R_ * S * C * 4
                table.append((p.data_ptr() + off, g.data_ptr() + off, k * R_ * S * C, 5e-4, plan, 1))
            op_src.append(p)
            n_op += n
        else:
            table.append((p, g, n, 5e-4, None, 0))
    n_all = sum(p.numel() for p in ps)
    torch.cuda.synchronize()
    res = {"case": "fused optimizer step, ResNet-18 table", "tensors": len(ps), "table_entries": len(table), "elements": n_all,
           "operand_elements": n_op, "gpu": gpu, "power_limit": power}
    for kind, kw, lr, per_el in (("sgd_momentum", dict(momentum=0.9), 0.1, 20), ("adamw", dict(betas=(0.9, 0.999), eps=1e-8), 1e-3, 28)):
        opt = pkg.FusedOptimizer(eng, pkg.OPTIM_SGD if kind.startswith("sgd") else pkg.OPTIM_ADAMW, table, **kw)
        ms = timed(lambda: opt.step(lr), iters)
        info = opt.info()
        opt.close()
        nbytes = per_el * n_all + 2 * n_op
        tp = [p.clone() for p in ps]
        for t, g in zip(tp, gs):
            t.grad = g
        topt = (torch.optim.SGD(tp, lr=lr, momentum=0.9, weight_decay=5e-4, fused=True) if kind.startswith("sgd")
                else torch.optim.AdamW(tp, lr=lr, weight_decay=5e-4, fused=True))
        ms_t = timed(topt.step, iters)
        res.update({f"{kind}_us": ms * 1e3, f"{kind}_bytes": nbytes, f"{kind}_GBps": nbytes / ms / 1e6,
                    f"{kind}_share_of_3350": nbytes / ms / 1e6 / HBM, f"{kind}_grid": info["grid"], f"{kind}_chunks": info["chunks"],
                    f"torch_fused_{kind}_us": ms_t * 1e3})
        del tp, topt
    bf = [torch.empty(p.numel(), dtype=torch.bfloat16, device="cuda") for p in op_src]
    res["torch_foreach_copy_bf16_us"] = timed(lambda: torch._foreach_copy_(bf, op_src), iters) * 1e3
    print(json.dumps(res), flush=True)
    for plan in plans:
        plan.close()


def run_resnetgap_optim(N, iters, rounds=3):
    """the GAP ResNet training step of run_resnetgap with every layer's sgd(lr) and with the fused SGD at momentum 0 (the same bits),
    alternated in this one call; then momentum SGD and AdamW.  The update alone (gradients left in place) is timed the same way."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from example_nets import ResNetGAP
    gpu, power = card()
    net = ResNetGAP(eng, pkg, ResNetGAP.init_params())
    xl = torch.randint(0, 0x3F80, (N * 28, 32), dtype=torch.int16, device="cuda")
    labels = torch.randint(0, 10, (N,), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    opts = {"fused_sgd": (pkg.SGD(eng, net.layers()), 0.2), "fused_sgd_momentum": (pkg.SGD(eng, net.layers(), momentum=0.9, weight_decay=5e-4), 0.02),
            "fused_adamw": (pkg.AdamW(eng, net.layers()), 1e-3)}
    updates = {"layer_sgd": lambda: net.sgd(0.2)}
    updates.update({k: (lambda o=o, lr=lr: o.step(lr)) for k, (o, lr) in opts.items()})

    def step(update):
        net.forward(xl.data_ptr(), labels)
        net.backward()
        update()

    out = {k: [] for k in updates}
    upd = {k: [] for k in updates}
    for _ in range(rounds):
        for k, u in updates.items():
            out[k].append(timed(lambda u=u: step(u), iters))
            upd[k].append(timed(u, iters))
    launches = {}
    for k, u in updates.items():
        n0 = eng.launch_count()
        u()
        launches[k] = eng.launch_count() - n0
    torch.cuda.synchronize()
    for o, _ in opts.values():
        o.close()
    net.close()
    print(json.dumps({"case": f"GAP ResNet training step N={N}, update variants alternated over {rounds} rounds",
                      "step_ms_median": {k: float(np.median(v)) for k, v in out.items()}, "step_ms_all": out,
                      "update_only_us_median": {k: float(np.median(v)) * 1e3 for k, v in upd.items()},
                      "kernel_launches_per_update": launches, "gpu": gpu, "power_limit": power}), flush=True)


def run_dwconv(name, N, H, W, C, R, stride, pad, iters):
    """the three passes of a depthwise convolution (pcnn_conv_tc_fwd on a DepthwiseConvPlan, pcnn_dwconv_dgrad, pcnn_dwconv_wgrad)
    next to F.conv2d(groups=C) and aten.convolution_backward on the same bf16 channels-last tensors.  Bytes per pass: x and y (or
    dy and dx, or x and dy) crossing HBM once, N (H W + P Q) C 2; the weight gradient adds its fp32 slots, written and read once,
    and dw."""
    info = pkg.dwconv_info(N, H, W, C, R, R, stride, (pad, pad))
    P, Q = info["P"], info["Q"]
    w = rng.uniform(-0.5, 0.5, (C, R, R)).astype(np.float32)
    plan = pkg.DepthwiseConvPlan(eng, N, H, W, C, R, R, w, None, act=0, stride=stride, padding=(pad, pad))
    bits = lambda *shape: torch.randint(0, 0x3F80, shape, dtype=torch.int16, device="cuda")
    x, dy = bits(N, H, W, C), bits(N, P, Q, C)
    y, dx = torch.empty((N, P, Q, C), dtype=torch.int16, device="cuda"), torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    dw = torch.empty((C, R, R), dtype=torch.float32, device="cuda")
    gpu, power = card()
    act_bytes = N * (H * W + P * Q) * C * 2
    slot_bytes = (2 * info["ranges"] * C * R * R * 4 if info["ranges"] > 1 else 0) + C * R * R * 4
    xt = x.view(torch.bfloat16).permute(0, 3, 1, 2)
    dyt = dy.view(torch.bfloat16).permute(0, 3, 1, 2)
    wt = torch.from_numpy(w).to("cuda").to(torch.bfloat16)[:, None].contiguous(memory_format=torch.channels_last)
    F = torch.nn.functional
    cb = torch.ops.aten.convolution_backward
    passes = (
        ("fwd", lambda: plan.fwd(x, y), lambda: F.conv2d(xt, wt, None, stride, pad, groups=C), act_bytes),
        ("dgrad", lambda: eng.dwconv_dgrad(plan, dy, dx),
         lambda: cb(dyt, xt, wt, None, [stride] * 2, [pad] * 2, [1, 1], False, [0, 0], C, [True, False, False]), act_bytes),
        ("wgrad", lambda: eng.dwconv_wgrad(plan, x, dy, dw),
         lambda: cb(dyt, xt, wt, None, [stride] * 2, [pad] * 2, [1, 1], False, [0, 0], C, [False, True, False]), act_bytes + slot_bytes),
    )
    for what, ours, theirs, nbytes in passes:
        ms, ms_torch = timed(ours, iters), timed(theirs, iters)
        print(json.dumps({"case": f"dwconv {name} {what}", "N": N, "us": ms * 1e3, "MB": nbytes / 1e6,
                          "share_of_3350": nbytes / (ms * 1e-3) / 1e9 / HBM, "torch_us": ms_torch * 1e3, "torch_over_ours": ms_torch / ms,
                          "vec": info["vec"], "wgrad_ranges": info["ranges"], "gpu": gpu, "power_limit": power}), flush=True)
    plan.close()


def run_mbblock(N, iters, k=3):
    """one training step of an inverted-residual block at 28x28x40, N = 128: 1x1 expand to 240 -> BN + ReLU -> depthwise k x k pad
    k // 2 -> BN + ReLU -> 1x1 project to 40 -> BN + x0, its backward (the shortcut's gradient dres left apart, as run_resblock)
    and the sgd of the six layers, on the engine's stream.  Next to it the torch eager step of the same block on bf16 channels-last
    tensors (fp32 masters, w -= lr * grad, re-cast to bf16)."""
    H = W = 28
    C, E = 40, 240
    r = np.random.default_rng(12)
    u = lambda shape, fan: r.uniform(-1, 1, shape).astype(np.float32) / np.float32(np.sqrt(fan))
    fe, fd, fp = u((E, 1, 1, C), C), u((E, k, k), k * k), u((C, 1, 1, E), E)
    ex = pkg.ConvLayer(eng, N, H, W, C, E, 1, 1, fe, None, act=0)
    dwl = pkg.DepthwiseConvLayer(eng, N, H, W, E, k, k, fd, None, act=0, padding=(k // 2, k // 2))
    pr = pkg.ConvLayer(eng, N, H, W, E, C, 1, 1, fp, None, act=0)
    b1, b2 = pkg.BatchNormLayer(eng, N, H, W, E, act=pkg.ACT_RELU), pkg.BatchNormLayer(eng, N, H, W, E, act=pkg.ACT_RELU)
    b3 = pkg.BatchNormLayer(eng, N, H, W, C, act=0)
    wide = lambda: torch.empty((N, H, W, E), dtype=torch.int16, device="cuda")
    narrow = lambda: torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    x0 = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    dout = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    dout ^= torch.randint(0, 2, (N, H, W, C), dtype=torch.int16, device="cuda") << 15
    ye, ze, yd, zd, dze, dye, dyd, dzd = (wide() for _ in range(8))
    yp, out, dyp, dres, dx0 = (narrow() for _ in range(5))
    lr = 0.05
    gpu, power = card()

    def step():
        ex.forward(x0, ye); b1.forward(ye, ze); dwl.forward(ze, yd); b2.forward(yd, zd); pr.forward(zd, yp); b3.forward(yp, out, r=x0)
        b3.backward(out, dout, dyp, dr=dres); pr.backward(yp, dyp, dzd); b2.backward(zd, dzd, dyd); dwl.backward(yd, dyd, dze)
        b1.backward(ze, dze, dye); ex.backward(ye, dye, dx0)
        for layer in (ex, b1, dwl, b2, pr, b3):
            layer.sgd(lr)

    ms = timed(step, iters)
    F = torch.nn.functional
    xt = x0.view(torch.bfloat16).permute(0, 3, 1, 2).detach().requires_grad_(True)
    dt = dout.view(torch.bfloat16).permute(0, 3, 1, 2)
    cl = lambda a: torch.from_numpy(a).to("cuda").contiguous(memory_format=torch.channels_last)
    m32 = {"fe": cl(fe.transpose(0, 3, 1, 2)), "fd": cl(fd[:, None]), "fp": cl(fp.transpose(0, 3, 1, 2))}
    for i, ch in ((1, E), (2, E), (3, C)):
        m32[f"g{i}"], m32[f"b{i}"] = torch.ones(ch, device="cuda"), torch.zeros(ch, device="cuda")
    mb = {kk: (v.to(torch.bfloat16) if kk.startswith("f") else v.clone()).requires_grad_(True) for kk, v in m32.items()}
    stats = [torch.zeros(ch, device="cuda") if j % 2 == 0 else torch.ones(ch, device="cuda") for ch in (E, E, C) for j in range(2)]

    def torch_step():
        for v in mb.values():
            v.grad = None
        xt.grad = None
        h = torch.relu(F.batch_norm(F.conv2d(xt, mb["fe"]), stats[0], stats[1], mb["g1"], mb["b1"], training=True))
        h = torch.relu(F.batch_norm(F.conv2d(h, mb["fd"], padding=k // 2, groups=E), stats[2], stats[3], mb["g2"], mb["b2"], training=True))
        h = F.batch_norm(F.conv2d(h, mb["fp"]), stats[4], stats[5], mb["g3"], mb["b3"], training=True) + xt
        h.backward(dt)
        with torch.no_grad():
            for kk in m32:
                m32[kk].add_(mb[kk].grad.float(), alpha=-lr)
                mb[kk].copy_(m32[kk])

    ms_torch = timed(torch_step, iters)
    ms_dw = {"fwd": timed(lambda: dwl.forward(ze, yd), iters), "bwd": timed(lambda: (eng.dwconv_wgrad(dwl.plan, ze, dyd, dwl.dw),
                                                                                      eng.dwconv_dgrad(dwl.plan, dyd, dze)), iters)}
    print(json.dumps({"case": f"inverted-residual block 28x28x40 -> 240 dw {k}x{k} training step N={N}", "ms": ms, "torch_eager_ms": ms_torch,
                      "ours_over_torch": ms / ms_torch, "dw_fwd_ms": ms_dw["fwd"], "dw_bwd_ms": ms_dw["bwd"], "families": [ex.family, pr.family],
                      "gpu": gpu, "power_limit": power}), flush=True)
    for layer in (ex, b1, dwl, b2, pr, b3):
        layer.close()


def run_gconv(name, N, H, W, C, K, G, R, stride, pad, iters):
    """the three passes of a grouped convolution (pcnn_conv_tc_fwd on a GroupedConvPlan, pcnn_gconv_dgrad, pcnn_gconv_wgrad) next
    to F.conv2d(groups=G) and aten.convolution_backward on the same bf16 channels-last tensors.  The bound of each pass is the larger
    of two times: bytes N (H W C + P Q K) 2 (x and y, or dy and dx, or x and dy crossing HBM once; the weight gradient adds its fp32
    slots, written and read once, and dw) over 3.35 TB/s, and 2 N P Q K Cg R S FLOPs over the 67 TFLOP/s fp32 data-sheet rate."""
    info = pkg.gconv_info(N, H, W, C, K, G, R, R, stride, (pad, pad))
    P, Q, Cg = info["P"], info["Q"], info["Cg"]
    w = rng.uniform(-0.5, 0.5, (K, R, R, Cg)).astype(np.float32)
    plan = pkg.GroupedConvPlan(eng, N, H, W, C, K, G, R, R, w, None, act=0, stride=stride, padding=(pad, pad))
    bits = lambda *shape: torch.randint(0, 0x3F80, shape, dtype=torch.int16, device="cuda")
    x, dy = bits(N, H, W, C), bits(N, P, Q, K)
    y, dx = torch.empty((N, P, Q, K), dtype=torch.int16, device="cuda"), torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    dw = torch.empty((K, R, R, Cg), dtype=torch.float32, device="cuda")
    gpu, power = card()
    act_bytes = N * (H * W * C + P * Q * K) * 2
    nw = K * R * R * Cg
    slot_bytes = (2 * info["ranges"] * nw * 4 if info["ranges"] > 1 else 0) + nw * 4
    flops = 2.0 * N * P * Q * K * Cg * R * R
    xt = x.view(torch.bfloat16).permute(0, 3, 1, 2)
    dyt = dy.view(torch.bfloat16).permute(0, 3, 1, 2)
    wt = torch.from_numpy(w).to("cuda").to(torch.bfloat16).permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
    F = torch.nn.functional
    cb = torch.ops.aten.convolution_backward
    passes = (
        ("fwd", lambda: plan.fwd(x, y), lambda: F.conv2d(xt, wt, None, stride, pad, groups=G), act_bytes),
        ("dgrad", lambda: eng.gconv_dgrad(plan, dy, dx),
         lambda: cb(dyt, xt, wt, None, [stride] * 2, [pad] * 2, [1, 1], False, [0, 0], G, [True, False, False]), act_bytes),
        ("wgrad", lambda: eng.gconv_wgrad(plan, x, dy, dw),
         lambda: cb(dyt, xt, wt, None, [stride] * 2, [pad] * 2, [1, 1], False, [0, 0], G, [False, True, False]), act_bytes + slot_bytes),
    )
    for what, ours, theirs, nbytes in passes:
        ms, ms_torch = timed(ours, iters), timed(theirs, iters)
        t_mem, t_flop = nbytes / (HBM * 1e9), flops / 67e12
        print(json.dumps({"case": f"gconv {name} {what}", "N": N, "us": ms * 1e3, "MB": nbytes / 1e6, "GFLOP": flops / 1e9,
                          "share_of_bound": max(t_mem, t_flop) / (ms * 1e-3), "bound": "HBM" if t_mem >= t_flop else "fp32",
                          "torch_us": ms_torch * 1e3, "torch_over_ours": ms_torch / ms, "Cg": Cg, "Kg": info["Kg"], "vec": info["vec"],
                          "kt": info["kt"], "wgrad_ranges": info["ranges"], "gpu": gpu, "power_limit": power}), flush=True)
    plan.close()


def run_resnextblock(N, iters):
    """one training step of a ResNeXt bottleneck at 56x56x256, N = 128: 1x1 reduce to 128 -> BN + ReLU -> grouped 3x3 pad 1, G = 32
    (Cg = 4) -> BN + ReLU -> 1x1 expand to 256 -> BN + x0 -> ReLU, its backward (the shortcut's gradient dres left apart, as
    run_resblock) and the sgd of the six layers, on the engine's stream.  Next to it the torch eager step of the same block on bf16
    channels-last tensors (fp32 masters, w -= lr * grad, re-cast to bf16)."""
    H = W = 56
    C, Dm, G = 256, 128, 32
    r = np.random.default_rng(13)
    u = lambda shape, fan: r.uniform(-1, 1, shape).astype(np.float32) / np.float32(np.sqrt(fan))
    fr, fg, fe = u((Dm, 1, 1, C), C), u((Dm, 3, 3, Dm // G), 9 * Dm // G), u((C, 1, 1, Dm), Dm)
    rd = pkg.ConvLayer(eng, N, H, W, C, Dm, 1, 1, fr, None, act=0)
    gl = pkg.GroupedConvLayer(eng, N, H, W, Dm, Dm, G, 3, 3, fg, None, act=0, padding=(1, 1))
    ex = pkg.ConvLayer(eng, N, H, W, Dm, C, 1, 1, fe, None, act=0)
    b1, b2 = pkg.BatchNormLayer(eng, N, H, W, Dm, act=pkg.ACT_RELU), pkg.BatchNormLayer(eng, N, H, W, Dm, act=pkg.ACT_RELU)
    b3 = pkg.BatchNormLayer(eng, N, H, W, C, act=pkg.ACT_RELU)
    mid = lambda: torch.empty((N, H, W, Dm), dtype=torch.int16, device="cuda")
    full = lambda: torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    x0 = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    dout = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    dout ^= torch.randint(0, 2, (N, H, W, C), dtype=torch.int16, device="cuda") << 15
    yr, zr, yg, zg, dzg, dyg, dzr, dyr = (mid() for _ in range(8))
    ye, out, dye, dres, dx0 = (full() for _ in range(5))
    lr = 0.05
    gpu, power = card()

    def step():
        rd.forward(x0, yr); b1.forward(yr, zr); gl.forward(zr, yg); b2.forward(yg, zg); ex.forward(zg, ye); b3.forward(ye, out, r=x0)
        b3.backward(out, dout, dye, dr=dres); ex.backward(ye, dye, dzg); b2.backward(zg, dzg, dyg); gl.backward(yg, dyg, dzr)
        b1.backward(zr, dzr, dyr); rd.backward(yr, dyr, dx0)
        for layer in (rd, b1, gl, b2, ex, b3):
            layer.sgd(lr)

    ms = timed(step, iters)
    F = torch.nn.functional
    xt = x0.view(torch.bfloat16).permute(0, 3, 1, 2).detach().requires_grad_(True)
    dt = dout.view(torch.bfloat16).permute(0, 3, 1, 2)
    cl = lambda a: torch.from_numpy(np.ascontiguousarray(a.transpose(0, 3, 1, 2))).to("cuda").contiguous(memory_format=torch.channels_last)
    m32 = {"fr": cl(fr), "fg": cl(fg), "fe": cl(fe)}
    for i, ch in ((1, Dm), (2, Dm), (3, C)):
        m32[f"g{i}"], m32[f"b{i}"] = torch.ones(ch, device="cuda"), torch.zeros(ch, device="cuda")
    mb = {kk: (v.to(torch.bfloat16) if kk.startswith("f") else v.clone()).requires_grad_(True) for kk, v in m32.items()}
    stats = [torch.zeros(ch, device="cuda") if j % 2 == 0 else torch.ones(ch, device="cuda") for ch in (Dm, Dm, C) for j in range(2)]

    def torch_step():
        for v in mb.values():
            v.grad = None
        xt.grad = None
        h = torch.relu(F.batch_norm(F.conv2d(xt, mb["fr"]), stats[0], stats[1], mb["g1"], mb["b1"], training=True))
        h = torch.relu(F.batch_norm(F.conv2d(h, mb["fg"], padding=1, groups=G), stats[2], stats[3], mb["g2"], mb["b2"], training=True))
        h = torch.relu(F.batch_norm(F.conv2d(h, mb["fe"]), stats[4], stats[5], mb["g3"], mb["b3"], training=True) + xt)
        h.backward(dt)
        with torch.no_grad():
            for kk in m32:
                m32[kk].add_(mb[kk].grad.float(), alpha=-lr)
                mb[kk].copy_(m32[kk])

    ms_torch = timed(torch_step, iters)
    ms_g = {"fwd": timed(lambda: gl.forward(zr, yg), iters), "bwd": timed(lambda: (eng.gconv_wgrad(gl.plan, zr, dyg, gl.dw),
                                                                                    eng.gconv_dgrad(gl.plan, dyg, dzr)), iters)}
    print(json.dumps({"case": f"ResNeXt bottleneck 56x56x256 -> 128 G{G} training step N={N}", "ms": ms, "torch_eager_ms": ms_torch,
                      "ours_over_torch": ms / ms_torch, "grouped_fwd_ms": ms_g["fwd"], "grouped_bwd_ms": ms_g["bwd"],
                      "families": [rd.family, ex.family], "gpu": gpu, "power_limit": power}), flush=True)
    for layer in (rd, b1, gl, b2, ex, b3):
        layer.close()


def run_se(name, N, H, W, C, iters):
    """the three squeeze-and-excitation passes (pcnn_se_scale_nhwc_bf16_fwd / _bwd_gate / _bwd_input) next to torch eager on the
    same bf16 channels-last tensors.  Bytes per pass, each [N][H][W][C] tensor crossing HBM once: forward x and y (plus r), gate
    x, dy, y read and g written plus its fp32 slots (written and read once) and ds, input gradient g and dx."""
    info = pkg.se_scale_nhwc_info(N, H, W, C)
    bits = lambda *shape: torch.randint(0, 0x3F80, shape, dtype=torch.int16, device="cuda") ^ (torch.randint(0, 2, shape, dtype=torch.int16, device="cuda") << 15)
    x, r, dy, y = (bits(N, H, W, C) for _ in range(4))
    g, dx = torch.empty_like(x), torch.empty_like(x)
    s = torch.rand((N, C), device="cuda").to(torch.bfloat16).view(torch.int16)
    pitch = (C + 7) // 8 * 8
    dpool, ds = bits(N, pitch), torch.empty((N, C), dtype=torch.int16, device="cuda")
    eng.se_scale_fwd(x, s, y, N, H, W, C, r=r, act=pkg.ACT_RELU)
    gpu, power = card()
    t = N * H * W * C * 2
    slot_bytes = 2 * N * info["ranges"] * C * 4 if info["ranges"] > 1 else 0
    cl = lambda a: a.view(torch.bfloat16).permute(0, 3, 1, 2)
    xt, rt, dyt, yt = cl(x), cl(r), cl(dy), cl(y)
    st, dpt = s.view(torch.bfloat16)[:, :, None, None], dpool.view(torch.bfloat16)[:, :C, None, None]
    passes = (
        ("fwd", lambda: eng.se_scale_fwd(x, s, y, N, H, W, C), lambda: xt * st, 2 * t),
        ("fwd + r + ReLU", lambda: eng.se_scale_fwd(x, s, y, N, H, W, C, r=r, act=pkg.ACT_RELU), lambda: torch.relu(xt * st + rt), 3 * t),
        ("gate (ReLU)", lambda: eng.se_scale_bwd_gate(x, y, dy, g, ds, N, H, W, C, act=pkg.ACT_RELU),
         lambda: (lambda gt: (gt, (gt * xt).sum((2, 3))))(torch.where(yt > 0, dyt, 0)), 4 * t + slot_bytes + N * C * 2),
        ("input + dpool", lambda: eng.se_scale_bwd_input(dy, s, dx, N, H, W, C, dpool=dpool, dpool_row_pitch=pitch),
         lambda: dyt * st + dpt / (H * W), 2 * t),
    )
    for what, ours, theirs, nbytes in passes:
        ms, ms_torch = timed(ours, iters), timed(theirs, iters)
        print(json.dumps({"case": f"se {name} {what}", "N": N, "us": ms * 1e3, "MB": nbytes / 1e6, "share_of_3350": nbytes / (ms * 1e-3) / 1e9 / HBM,
                          "torch_us": ms_torch * 1e3, "torch_over_ours": ms_torch / ms, "vec": info["vec"], "gate_ranges": info["ranges"],
                          "gate_ctas": info["ctas"], "gpu": gpu, "power_limit": power}), flush=True)


def run_seblock(N, iters, hid=8):
    """one training step of an SE basic block, 56x56x64 at N = 128: conv_a 3x3 pad 1 -> BN + ReLU -> conv_b -> BN -> SE (64 -> hid ->
    64, hid 8: the smallest width the linear row pitch allows, where SE-ResNet's reduction 16 would give 4) carrying + x0 and the
    ReLU, its backward (dx0 and the shortcut's gradient dres left apart, as run_resblock) and the sgd of the five layers, on the
    engine's stream.  Next to it the torch eager step of the same block on bf16 channels-last tensors (fp32 masters, w -= lr * grad,
    re-cast to bf16)."""
    H = W = 56
    C = 64
    r = np.random.default_rng(13)
    u = lambda shape, fan: r.uniform(-1, 1, shape).astype(np.float32) / np.float32(np.sqrt(fan))
    fa, fb = u((C, 3, 3, C), 9 * C), u((C, 3, 3, C), 9 * C)
    w1, b1, w2, b2 = u((hid, C), C), u(hid, C), u((C, hid), hid), u(C, hid)
    ca = pkg.ConvLayer(eng, N, H, W, C, C, 3, 3, fa, None, act=0, padding=(1, 1))
    cb = pkg.ConvLayer(eng, N, H, W, C, C, 3, 3, fb, None, act=0, padding=(1, 1))
    ba, bb = pkg.BatchNormLayer(eng, N, H, W, C, act=pkg.ACT_RELU), pkg.BatchNormLayer(eng, N, H, W, C, act=0)
    se = pkg.SqueezeExcitationLayer(eng, N, H, W, C, hid, w1, b1, w2, b2, act=pkg.ACT_RELU)
    e = lambda: torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    x0 = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    dout = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    dout ^= torch.randint(0, 2, (N, H, W, C), dtype=torch.int16, device="cuda") << 15
    ya, za, yb, zb, out, dzb, dyb, dres, dza, dya, dx0 = (e() for _ in range(11))
    lr = 0.05
    gpu, power = card()

    def step():
        ca.forward(x0, ya); ba.forward(ya, za); cb.forward(za, yb); bb.forward(yb, zb); se.forward(zb, out, r=x0)
        se.backward(out, dout, dzb, dr=dres); bb.backward(zb, dzb, dyb); cb.backward(yb, dyb, dza); ba.backward(za, dza, dya)
        ca.backward(ya, dya, dx0)
        for layer in (ca, ba, cb, bb, se):
            layer.sgd(lr)

    ms = timed(step, iters)
    ms_se = {"fwd": timed(lambda: se.forward(zb, out, r=x0), iters), "bwd": timed(lambda: se.backward(out, dout, dzb, dr=dres), iters)}
    F = torch.nn.functional
    xt = x0.view(torch.bfloat16).permute(0, 3, 1, 2).detach().requires_grad_(True)
    dt = dout.view(torch.bfloat16).permute(0, 3, 1, 2)
    m32 = {k: torch.from_numpy(v).to("cuda").permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last) for k, v in
           (("fa", fa), ("fb", fb))}
    m32.update(ga=torch.ones(C, device="cuda"), ba=torch.zeros(C, device="cuda"), gb=torch.ones(C, device="cuda"), bb=torch.zeros(C, device="cuda"))
    m32.update({k: torch.from_numpy(v).to("cuda") for k, v in (("w1", w1), ("b1", b1), ("w2", w2), ("b2", b2))})
    mb = {k: (v.to(torch.bfloat16) if k[0] in "fwb" and k not in ("ba", "bb") else v.clone()).requires_grad_(True) for k, v in m32.items()}
    stats = [torch.zeros(C, device="cuda"), torch.ones(C, device="cuda"), torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")]

    def torch_step():
        for v in mb.values():
            v.grad = None
        xt.grad = None
        h = torch.relu(F.batch_norm(F.conv2d(xt, mb["fa"], padding=1), stats[0], stats[1], mb["ga"], mb["ba"], training=True))
        h = F.batch_norm(F.conv2d(h, mb["fb"], padding=1), stats[2], stats[3], mb["gb"], mb["bb"], training=True)
        s = torch.sigmoid(F.linear(torch.relu(F.linear(h.mean((2, 3)), mb["w1"], mb["b1"])), mb["w2"], mb["b2"]))
        h = torch.relu(h * s[:, :, None, None] + xt)
        h.backward(dt)
        with torch.no_grad():
            for k in m32:
                m32[k].add_(mb[k].grad.float(), alpha=-lr)
                mb[k].copy_(m32[k])

    ms_torch = timed(torch_step, iters)
    print(json.dumps({"case": f"SE basic block 56x56x64 (SE 64 -> {hid} -> 64) training step N={N}", "ms": ms, "torch_eager_ms": ms_torch,
                      "ours_over_torch": ms / ms_torch, "se_fwd_ms": ms_se["fwd"], "se_bwd_ms": ms_se["bwd"], "gpu": gpu,
                      "power_limit": power}), flush=True)
    for layer in (ca, cb, ba, bb, se):
        layer.close()


def run_bnact(name, N, H, W, C, iters, rounds=3):
    """batch normalization followed by ReLU (3), SiLU (4), hard-swish (5) or ReLU6 (6): training forward, eval forward and backward
    (pcnn_batchnorm_nhwc_bf16_bwd at 3, pcnn_batchnorm_nhwc_bf16_bwd_preact at 4-6), each with and without the residual r, the
    codes alternated over `rounds` rounds (the best of each kept), next to torch's F.batch_norm (+ add) + relu / silu / hardswish /
    relu6 and its autograd backward on the same channels-last bf16 tensors.  Bytes, T = N*H*W*C*2: the forwards as run_bn; the
    backward 7T at code 3 (x, y, dy read twice, dx written) and 5T at 4-6 (x, dy read twice, dx written), + 2T for reading r twice
    at 4-6, + T for writing dr."""
    M = N * H * W
    T = M * C * 2
    rnd = lambda: torch.randint(-0x4000, 0x4000, (M, C), dtype=torch.int16, device="cuda") & 0x3FFF | 0x3C00   # bf16 in [1, 2) * 2^k
    x, r, dy = rnd(), rnd(), rnd()
    r ^= torch.randint(0, 2, (M, C), dtype=torch.int16, device="cuda") << 15
    dy ^= torch.randint(0, 2, (M, C), dtype=torch.int16, device="cuda") << 15
    y, dx, dr = (torch.empty((M, C), dtype=torch.int16, device="cuda") for _ in range(3))
    info = pkg.batchnorm_nhwc_info(M, C)
    f = lambda v: eng.to_device(np.full(C, v, np.float32))
    gamma, beta, rm, rv, sm, sr, dg, db = f(1), f(0), f(0), f(1), f(0), f(1), f(0), f(0)
    gpu, power = card()
    F = torch.nn.functional
    acts = {3: torch.relu, 4: F.silu, 5: F.hardswish, 6: F.relu6}
    bf = lambda t: t.view(torch.bfloat16).reshape(N, H, W, C).permute(0, 3, 1, 2)         # channels-last NCHW views
    xt, rt, dyt = bf(x).detach().clone().requires_grad_(True), bf(r).detach().clone().requires_grad_(True), bf(dy)
    gt, bt = torch.ones(C, device="cuda", requires_grad=True), torch.zeros(C, device="cuda", requires_grad=True)
    rmt, rvt = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")

    def torch_fwd(act, with_r, training):
        v = F.batch_norm(xt, rmt, rvt, gt, bt, training=training, momentum=0.1, eps=1e-5)
        return acts[act](v + rt if with_r else v)

    def ours_bwd(act, rr, drr):
        if act == 3:
            return eng.batchnorm_bwd(x, y, dy, gamma, sm, sr, dx, dg, db, M, C, act=3, dr=drr)
        return eng.batchnorm_bwd_preact(x, dy, gamma, beta, sm, sr, dx, dg, db, M, C, act, r=rr, dr=drr)

    for with_r in (False, True):
        rr, drr = (r, dr) if with_r else (None, None)
        ins = [xt, gt, bt] + ([rt] if with_r else [])
        outs = {a: torch_fwd(a, with_r, True) for a in acts}
        best = {}
        for _ in range(rounds):
            for act in acts:
                eng.batchnorm_fwd(x, y, M, C, gamma, beta, rm, rv, sm, sr, r=rr, act=act)      # warm the training forward's path
                # the backward right after the training forward, so that at act 3 it reads that forward's y
                passes = (("training fwd", lambda: eng.batchnorm_fwd(x, y, M, C, gamma, beta, rm, rv, sm, sr, r=rr, act=act),
                           lambda: torch_fwd(act, with_r, True), 3 * T + (T if with_r else 0)),
                          ("bwd", lambda: ours_bwd(act, rr, drr), lambda: torch.autograd.grad(outs[act], ins, dyt, retain_graph=True),
                           (7 * T if act == 3 else 5 * T + (2 * T if with_r else 0)) + (T if with_r else 0)),
                          ("eval fwd", lambda: eng.batchnorm_fwd(x, y, M, C, gamma, beta, rm, rv, r=rr, act=act, training=False),
                           lambda: torch_fwd(act, with_r, False), 2 * T + (T if with_r else 0)))
                for what, fn, tfn, nbytes in passes:
                    ms, ms_torch = timed(fn, iters), timed(tfn, iters)
                    old = best.get((act, what))
                    best[(act, what)] = (min(ms, old[0]) if old else ms, min(ms_torch, old[1]) if old else ms_torch, nbytes)
        for what in ("training fwd", "eval fwd", "bwd"):
            ms3 = best[(3, what)][0]
            for act in acts:
                ms, ms_torch, nbytes = best[(act, what)]
                print(json.dumps({"case": f"{name} {what}" + (" + r" if with_r else ""), "act": act, "N": N, "us": ms * 1e3, "MB": nbytes / 1e6,
                                  "hbm_frac": nbytes / (ms * 1e-3) / 1e9 / HBM, "over_act3": ms / ms3, "torch_us": ms_torch * 1e3,
                                  "torch_over_ours": ms_torch / ms, "vec": info["vec"], "gpu": gpu, "power_limit": power}), flush=True)
    for a in (gamma, beta, rm, rv, sm, sr, dg, db):
        a.free()
    del x, r, dy, y, dx, dr, xt, rt


def run_gn(name, N, H, W, C, G, iters, rounds=3):
    """group normalization: the forward at ReLU without and with the residual r, the backward at ReLU (pcnn_groupnorm_nhwc_bf16_bwd,
    with dr) and, at SiLU with r, the forward and the pre-activation backward with dr (pcnn_groupnorm_nhwc_bf16_bwd_preact), the
    passes alternated over `rounds` rounds (the best of each kept), next to torch's F.group_norm (+ add) + relu / silu and its
    autograd backward on the same channels-last bf16 tensors.  Bytes, T = N*H*W*C*2: forward 3T (x read twice, y written) + T for
    r; backward at ReLU 7T (x, y, dy read twice, dx written) + T for dr; at SiLU 7T (x, r, dy read twice, dx written) + T for dr."""
    HW = H * W
    T = N * HW * C * 2
    rnd = lambda: torch.randint(-0x4000, 0x4000, (N * HW, C), dtype=torch.int16, device="cuda") & 0x3FFF | 0x3C00   # bf16 in [1, 2) * 2^k
    x, r, dy = rnd(), rnd(), rnd()
    r ^= torch.randint(0, 2, (N * HW, C), dtype=torch.int16, device="cuda") << 15
    dy ^= torch.randint(0, 2, (N * HW, C), dtype=torch.int16, device="cuda") << 15
    y, dx, dr = (torch.empty((N * HW, C), dtype=torch.int16, device="cuda") for _ in range(3))
    info = pkg.groupnorm_nhwc_info(N, HW, C, G)
    f = lambda v, n: eng.to_device(np.full(n, v, np.float32))
    gamma, beta, dg, db = f(1, C), f(0, C), f(0, C), f(0, C)
    sm, sr, ds = f(0, N * G), f(1, N * G), f(0, 2 * N * G)
    gpu, power = card()
    F = torch.nn.functional
    bf = lambda t: t.view(torch.bfloat16).reshape(N, H, W, C).permute(0, 3, 1, 2)         # channels-last NCHW views
    xt, rt, dyt = bf(x).detach().clone().requires_grad_(True), bf(r).detach().clone().requires_grad_(True), bf(dy)
    gt = torch.ones(C, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    bt = torch.zeros(C, device="cuda", dtype=torch.bfloat16, requires_grad=True)

    def torch_fwd(act, with_r):
        v = F.group_norm(xt, G, gt, bt, 1e-5)
        return act(v + rt if with_r else v)

    out_relu, out_silu = torch_fwd(torch.relu, True), torch_fwd(F.silu, True)
    passes = (("fwd", lambda: eng.groupnorm_fwd(x, y, N, HW, C, G, gamma, beta, sm, sr, act=3), lambda: torch_fwd(torch.relu, False), 3 * T),
              ("fwd + r", lambda: eng.groupnorm_fwd(x, y, N, HW, C, G, gamma, beta, sm, sr, r=r, act=3), lambda: torch_fwd(torch.relu, True),
               4 * T),
              ("bwd + dr", lambda: eng.groupnorm_bwd(x, y, dy, gamma, sm, sr, dx, dg, db, ds, N, HW, C, G, act=3, dr=dr),
               lambda: torch.autograd.grad(out_relu, [xt, gt, bt, rt], dyt, retain_graph=True), 8 * T),
              ("SiLU fwd + r", lambda: eng.groupnorm_fwd(x, y, N, HW, C, G, gamma, beta, sm, sr, r=r, act=4), lambda: torch_fwd(F.silu, True),
               4 * T),
              ("SiLU preact bwd + dr", lambda: eng.groupnorm_bwd_preact(x, dy, gamma, beta, sm, sr, dx, dg, db, ds, N, HW, C, G, 4, r=r, dr=dr),
               lambda: torch.autograd.grad(out_silu, [xt, gt, bt, rt], dyt, retain_graph=True), 8 * T))
    best = {}
    for _ in range(rounds):
        for what, fn, tfn, nbytes in passes:
            ms, ms_torch = timed(fn, iters), timed(tfn, iters)
            old = best.get(what)
            best[what] = (min(ms, old[0]) if old else ms, min(ms_torch, old[1]) if old else ms_torch, nbytes)
    for what, _, _, _ in passes:
        ms, ms_torch, nbytes = best[what]
        print(json.dumps({"case": f"{name} {what}", "N": N, "G": G, "us": ms * 1e3, "MB": nbytes / 1e6,
                          "hbm_frac": nbytes / (ms * 1e-3) / 1e9 / HBM, "torch_us": ms_torch * 1e3, "torch_over_ours": ms_torch / ms,
                          "vec": info["vec"], "ranges": info["ranges"], "ctas": info["ctas"], "gpu": gpu, "power_limit": power}), flush=True)
    for a in (gamma, beta, dg, db, sm, sr, ds):
        a.free()
    del x, r, dy, y, dx, dr, xt, rt


def run_dropout(name, N, H, W, C, iters, per_sample, p=0.2, rounds=3):
    """dropout (element mode) or stochastic depth with r (per-sample mode) at p: the forward and the backward (the same call on dy,
    without r), ours and torch's alternated over `rounds` rounds (the best of each kept), on the same bf16 channels-last tensors.
    torch: F.dropout and aten.native_dropout_backward, which write and read a bool mask; for stochastic depth the eager
    x * bernoulli(N, 1, 1, 1) / (1 - p) + r and dy * that multiplier.  Bytes, T = N*H*W*C*2: ours 2T each way, + T for r; torch's
    element mode T / 2 more each way (the mask)."""
    E = H * W * C
    T = N * E * 2
    rnd = lambda: torch.randint(-0x4000, 0x4000, (N, E), dtype=torch.int16, device="cuda") & 0x3FFF | 0x3C00   # bf16 in [1, 2) * 2^k
    x, r, dy = rnd(), rnd(), rnd()
    y, dx = torch.empty_like(x), torch.empty_like(x)
    gpu, power = card()
    F = torch.nn.functional
    bf = lambda t: t.view(torch.bfloat16).reshape(N, H, W, C).permute(0, 3, 1, 2)         # channels-last NCHW views
    xt, rt, dyt = bf(x), bf(r), bf(dy)
    rr = r if per_sample else None
    calls = iter(range(1, 1 << 40))
    ours = {"fwd": lambda: eng.dropout(x, y, N, E, p, 1, next(calls), per_sample, r=rr),
            "bwd": lambda: eng.dropout(dy, dx, N, E, p, 1, 7, per_sample)}
    if per_sample:
        m = torch.empty((N, 1, 1, 1), dtype=torch.bfloat16, device="cuda").bernoulli_(1 - p).div_(1 - p)
        theirs = {"fwd": lambda: xt * torch.empty((N, 1, 1, 1), dtype=torch.bfloat16, device="cuda").bernoulli_(1 - p).div_(1 - p) + rt,
                  "bwd": lambda: dyt * m}
        nbytes = {"fwd": 3 * T, "bwd": 2 * T}
        torch_bytes = nbytes
    else:
        _, mask = torch.ops.aten.native_dropout(xt, p, True)
        theirs = {"fwd": lambda: F.dropout(xt, p, training=True),
                  "bwd": lambda: torch.ops.aten.native_dropout_backward(dyt, mask, 1.0 / (1.0 - p))}
        nbytes = {"fwd": 2 * T, "bwd": 2 * T}
        torch_bytes = {k: v + T // 2 for k, v in nbytes.items()}
    info = pkg.dropout_info(N, E, 0, p, per_sample)
    best = {}
    for _ in range(rounds):
        for what in ("fwd", "bwd"):
            ms, ms_torch = timed(ours[what], iters), timed(theirs[what], iters)
            old = best.get(what, (ms, ms_torch))
            best[what] = (min(ms, old[0]), min(ms_torch, old[1]))
    for what in ("fwd", "bwd"):
        ms, ms_torch = best[what]
        print(json.dumps({"case": f"{'stochastic depth + r' if per_sample else 'dropout'} {name} {what}", "N": N, "p": p, "us": ms * 1e3,
                          "MB": nbytes[what] / 1e6, "hbm_frac": nbytes[what] / (ms * 1e-3) / 1e9 / HBM, "torch_us": ms_torch * 1e3,
                          "torch_hbm_frac": torch_bytes[what] / (ms_torch * 1e-3) / 1e9 / HBM, "torch_over_ours": ms_torch / ms,
                          "vec": info["vec"], "grid": info["grid"], "gpu": gpu, "power_limit": power}), flush=True)
    del x, r, dy, y, dx


def run_augment(name, N, H, W, C, C_out, pad, iters, batches=4, row_pitch=0, image_rows=0, rounds=3):
    """one batch of the input pipeline (pcnn_augment_u8_bf16): shuffle over a dataset of `batches` batches, crop with pad, flip,
    normalise, into x with C_out channels; the calls walk the epoch's batches.  Beside it the torch eager pipeline of
    tests/augment_ref.py (torch_batch: gather, pad, crop and flip by advanced indexing, normalise, cast) on the same indices,
    offsets and flips, plus the label gather, alternated over `rounds` rounds (the best of each kept).  Bytes: N H W C read,
    N H W C_out 2 written, 2 N for the labels."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import augment_ref as A
    n = N * batches
    images = torch.randint(0, 256, (n, H, W, C), dtype=torch.uint8, device="cuda")
    labels = torch.randint(0, 10, (n,), dtype=torch.uint8, device="cuda")
    flip = True
    mean, std = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)) if C == 3 else (None, None)
    info, _ = pkg.augment_info(n, H, W, C, 0, N, 1, pad, int(flip), C_out, row_pitch, image_rows, mean, std)
    x = torch.empty(N * info["image_rows"] * info["row_pitch"], dtype=torch.int16, device="cuda")
    lo = torch.empty(N, dtype=torch.uint8, device="cuda")
    steps = iter(range(1 << 40))
    seed, epoch = 11, 3

    def ours():
        eng.augment(images, labels, n, H, W, C, (next(steps) % batches) * N, N, x, lo, shuffle=1, pad=pad, flip=int(flip), seed=seed,
                    epoch=epoch, mean=mean, std=std, C_out=C_out, row_pitch=row_pitch, image_rows=image_rows)

    draws = []
    for b in range(batches):
        i = A.indices(n, b * N, N, 1, seed, epoch)
        oy, ox, fl = A.draws(i.astype(np.uint64), pad, int(flip), seed, epoch)
        draws.append([torch.as_tensor(a, device="cuda") for a in (i, oy, ox, fl)])
    tsteps = iter(range(1 << 40))

    def theirs():
        i, oy, ox, fl = draws[next(tsteps) % batches]
        return A.torch_batch(images, i, oy, ox, fl, pad, mean, std, C_out), labels[i]

    gpu, power = card()
    best = None
    for _ in range(rounds):
        ms, ms_torch = timed(ours, iters), timed(theirs, iters)
        best = (ms, ms_torch) if best is None else (min(ms, best[0]), min(ms_torch, best[1]))
    ms, ms_torch = best
    nbytes = N * H * W * C + N * H * W * C_out * 2 + 2 * N
    print(json.dumps({"case": f"augment {name}", "N": N, "n": n, "pad": pad, "flip": flip, "us": ms * 1e3, "MB": nbytes / 1e6,
                      "hbm_frac": nbytes / (ms * 1e-3) / 1e9 / HBM, "torch_us": ms_torch * 1e3, "torch_over_ours": ms_torch / ms,
                      "vec": info["vec"], "grid": info["grid"], "rows_per_cta": info["rows_per_cta"], "gpu": gpu, "power_limit": power}),
          flush=True)


def run_augment_mix(name, N, H, W, C, C_out, pad, iters, batches=4, row_pitch=0, image_rows=0, rounds=3):
    """one mixed batch (pcnn_augment_mix_u8_bf16) in each mode against the plain batch (pcnn_augment_u8_bf16) of the same shape,
    and torchvision's v2.MixUp / v2.CutMix on torch's eager fp32 batch (tests/mix_ref.py's torch_f32_batch, then the cast),
    alternated over `rounds` rounds (the best of each kept).  Bytes: MixUp reads 2 N H W C, CutMix and the plain call N H W C;
    each writes N H W C_out 2."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import augment_ref as A
    from mix_ref import torch_f32_batch
    from torchvision.transforms import v2
    n = N * batches
    images = torch.randint(0, 256, (n, H, W, C), dtype=torch.uint8, device="cuda")
    labels = torch.randint(0, 10, (n,), dtype=torch.uint8, device="cuda")
    mean, std = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)) if C == 3 else (None, None)
    info, _ = pkg.augment_info(n, H, W, C, 0, N, 1, pad, 1, C_out, row_pitch, image_rows, mean, std)
    x = torch.empty(N * info["image_rows"] * info["row_pitch"], dtype=torch.int16, device="cuda")
    lo, lb = torch.empty(N, dtype=torch.uint8, device="cuda"), torch.empty(N, dtype=torch.uint8, device="cuda")
    steps = iter(range(1 << 40))
    seed, epoch, lam = 11, 3, 0.37
    box = (W // 4, H // 4, W - W // 4, H - H // 4)
    kw = dict(shuffle=1, pad=pad, flip=1, seed=seed, epoch=epoch, mean=mean, std=std, C_out=C_out, row_pitch=row_pitch,
              image_rows=image_rows)
    first = lambda: (next(steps) % batches) * N
    plain = lambda: eng.augment(images, labels, n, H, W, C, first(), N, x, lo, **kw)
    mix = {mode: (lambda mode=mode: eng.augment_mix(images, labels, n, H, W, C, first(), N, x, lo, lb, mode=mode, lam=lam, box=box, **kw))
           for mode in (pkg.MIX_MIXUP, pkg.MIX_CUTMIX)}
    draws = []
    for b in range(batches):
        i = A.indices(n, b * N, N, 1, seed, epoch)
        oy, ox, fl = A.draws(i.astype(np.uint64), pad, 1, seed, epoch)
        draws.append((i, oy, ox, fl))
    tv = {pkg.MIX_MIXUP: v2.MixUp(alpha=1.0, num_classes=10), pkg.MIX_CUTMIX: v2.CutMix(alpha=1.0, num_classes=10)}
    tv[pkg.MIX_MIXUP].make_params = lambda flat: dict(lam=lam)
    tv[pkg.MIX_CUTMIX].make_params = lambda flat: dict(box=box, lam_adjusted=lam)
    tsteps = iter(range(1 << 40))

    def theirs(mode):
        i, oy, ox, fl = draws[next(tsteps) % batches]
        out, y = tv[mode](torch_f32_batch(images, i, oy, ox, fl, pad, mean, std), labels[torch.as_tensor(i, device="cuda")].long())
        return out.permute(0, 2, 3, 1).to(torch.bfloat16), y

    gpu, power = card()
    for mode, kind in ((pkg.MIX_MIXUP, "MixUp"), (pkg.MIX_CUTMIX, "CutMix")):
        best = None
        for _ in range(rounds):
            r = (timed(mix[mode], iters), timed(plain, iters), timed(lambda: theirs(mode), iters))
            best = r if best is None else tuple(min(a, b) for a, b in zip(r, best))
        ms, ms_plain, ms_torch = best
        nbytes = N * H * W * C * (2 if mode == pkg.MIX_MIXUP else 1) + N * H * W * C_out * 2 + 3 * N
        print(json.dumps({"case": f"augment-mix {kind} {name}", "N": N, "n": n, "pad": pad, "us": ms * 1e3, "plain_us": ms_plain * 1e3,
                          "mix_over_plain": ms / ms_plain, "MB": nbytes / 1e6, "hbm_frac": nbytes / (ms * 1e-3) / 1e9 / HBM,
                          "torchvision_us": ms_torch * 1e3, "torchvision_over_ours": ms_torch / ms, "vec": info["vec"], "grid": info["grid"],
                          "gpu": gpu, "power_limit": power}), flush=True)


def run_resnetgap_mix(iters, rounds=3):
    """one training step of the GAP ResNet at N = 128 fed by pkg.ImageBatcher with shuffle, pad 2, mixup_alpha 0.2 and
    cutmix_alpha 1.0 and trained against the soft target (label smoothing 0.1), against the same step on the plain batcher with the
    hard loss, alternated over `rounds` rounds (the best of each kept)"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from example_nets import ResNetGAP

    class MixedResNetGAP(ResNetGAP):                                   # the soft loss over the network's z, as test_mix_gpu's
        def forward(self, x, t, training=True):
            super().forward(x, t.labels, training)
            self.eng.softmax_ce_soft_bf16(self.z, t.labels, self.NB, 10, 1.0 / self.NB, self.dz, self.loss, self.pred, labels_b=t.labels_b,
                                          lam=t.lam, smoothing=0.1)
    g = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    make = lambda **k: pkg.ImageBatcher(eng, g["train_u8"].reshape(-1, 28, 28), g["train_labels"], ResNetGAP.NB, pad=2, shuffle=True,
                                        seed=5, row_pitch=32, image_rows=28, **k)
    plain_b, mix_b = make(), make(mixup_alpha=0.2, cutmix_alpha=1.0)
    plain_net, mix_net = ResNetGAP(eng, pkg, ResNetGAP.init_params()), MixedResNetGAP(eng, pkg, ResNetGAP.init_params())
    k = iter(range(1 << 40))

    def step(net, batcher):
        net.forward(*batcher.batch(next(k) % batcher.steps_per_epoch))
        net.backward()
        net.sgd(ResNetGAP.LR_STEP)

    gpu, power = card()
    best = None
    for _ in range(rounds):
        r = (timed(lambda: step(mix_net, mix_b), iters), timed(lambda: step(plain_net, plain_b), iters))
        best = r if best is None else tuple(min(a, b) for a, b in zip(r, best))
    ms_mix, ms_plain = best
    print(json.dumps({"case": f"GAP ResNet training step N={ResNetGAP.NB}, mixed batch + soft loss vs plain batch + hard loss",
                      "ms_mix": ms_mix, "ms_plain": ms_plain, "mix_over_plain": ms_mix / ms_plain, "gpu": gpu, "power_limit": power}),
          flush=True)
    for a in (plain_b, mix_b, plain_net, mix_net):
        a.close()


def run_resnetgap_augment(iters, rounds=3):
    """one training step of the GAP ResNet of tests/example_nets.py at N = 128 on the 1024 golden digits, its batch built
    by pkg.ImageBatcher (shuffle, random crop of pad 2) against the same step on a slice of the pre-converted mnist_device rows,
    alternated over `rounds` rounds (the best of each kept)"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from example_nets import ResNetGAP, Slices
    g = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    slices = Slices(pkg, g["train_u8"], g["train_labels"], ResNetGAP.NB)
    net = ResNetGAP(eng, pkg, ResNetGAP.init_params())
    batcher = pkg.ImageBatcher(eng, g["train_u8"].reshape(-1, 28, 28), g["train_labels"], ResNetGAP.NB, pad=2, shuffle=True, seed=5,
                               row_pitch=32, image_rows=28)
    k = iter(range(1 << 40))

    def step(batch):
        s = next(k) % batcher.steps_per_epoch
        net.forward(*batch(s))
        net.backward()
        net.sgd(ResNetGAP.LR_STEP)

    aug = lambda: step(batcher.batch)
    plain = lambda: step(slices.batch)
    batch_only = lambda: batcher.batch(next(k) % batcher.steps_per_epoch)
    gpu, power = card()
    best = None
    for _ in range(rounds):
        r = (timed(aug, iters), timed(plain, iters), timed(batch_only, iters))
        best = r if best is None else tuple(min(a, b) for a, b in zip(r, best))
    ms_aug, ms_plain, ms_batch = best
    print(json.dumps({"case": f"GAP ResNet training step N={ResNetGAP.NB}, batch from ImageBatcher (shuffle, pad 2) vs pre-converted slice",
                      "ms_batcher": ms_aug, "ms_slice": ms_plain, "batcher_over_slice": ms_aug / ms_plain, "batch_us": ms_batch * 1e3,
                      "gpu": gpu, "power_limit": power}), flush=True)
    batcher.close()
    net.close()


def run_resized(name, N, H, W, C, H_out, W_out, C_out, iters, resize_size, batches=4, row_pitch=0, image_rows=0, rounds=3):
    """one resized batch (pcnn_augment_resized_u8_bf16) in each mode, RandomResizedCrop (default scale and ratio) + flip and
    Resize(resize_size) + CenterCrop, against the plain batch (pcnn_augment_u8_bf16, pad 0, flip) of the same output size from a
    dataset of that size, alternated over `rounds` rounds (the best of each kept); and torchvision's per-image CPU path for the same
    batch (resized_crop or resize + center_crop, flip, ToTensor + Normalize, bf16), which a data loader would otherwise run, timed
    once.  Bytes: the source bytes the boxes (or the eval window's preimage) cover, plus N H_out W_out C_out 2 written."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import resize_ref as RR
    import torchvision.transforms.v2.functional as TF
    n = N * batches
    images = torch.randint(0, 256, (n, H, W, C), dtype=torch.uint8, device="cuda")
    small = torch.randint(0, 256, (n, H_out, W_out, C), dtype=torch.uint8, device="cuda")
    labels = torch.randint(0, 10, (n,), dtype=torch.uint8, device="cuda")
    mean, std = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)) if C == 3 else (None, None)
    info, _ = pkg.augment_resized_info(n, H, W, C, 0, N, H_out, W_out, C_out=C_out, row_pitch=row_pitch, image_rows=image_rows)
    x = torch.empty(N * info["image_rows"] * info["row_pitch"], dtype=torch.int16, device="cuda")
    lo = torch.empty(N, dtype=torch.uint8, device="cuda")
    steps = iter(range(1 << 40))
    seed, epoch = 11, 3
    kw = dict(flip=1, seed=seed, epoch=epoch, mean=mean, std=std, C_out=C_out, row_pitch=row_pitch, image_rows=image_rows)
    first = lambda: (next(steps) % batches) * N
    calls = {m: (lambda m=m: eng.augment_resized(images, labels, n, H, W, C, first(), N, x, H_out, W_out, lo, mode=m, shuffle=int(m == 1),
                                                 resize_size=resize_size, **kw)) for m in (pkg.RESIZE_TRAIN, pkg.RESIZE_EVAL)}
    plain = lambda: eng.augment(small, labels, n, H_out, W_out, C, first(), N, x, lo, shuffle=1, pad=0, **kw)
    host = images[:N].cpu().permute(0, 3, 1, 2).contiguous()
    i = RR.A.indices(n, 0, N, 1, seed, epoch)
    box = np.stack(RR.boxes(i.astype(np.uint64), H, W, (0.08, 1.0), (3 / 4, 4 / 3), seed, epoch)[:4], -1)
    Rh, Rw = RR.resized_size(H, W, resize_size)
    m_t = torch.tensor(mean or (0.0,) * C).view(-1, 1, 1)
    s_t = torch.tensor(std or (1.0,) * C).view(-1, 1, 1)

    def torchvision_cpu(mode):
        t0 = time.perf_counter()
        for j in range(N):
            if mode == pkg.RESIZE_TRAIN:
                t, l, h, w = (int(v) for v in box[j])
                u = TF.horizontal_flip(TF.resized_crop(host[j], t, l, h, w, [H_out, W_out], antialias=True))
            else:
                u = TF.center_crop(TF.resize(host[j], resize_size, antialias=True), [H_out, W_out])
            ((u.float() / 255.0 - m_t) / s_t).to(torch.bfloat16)
        return time.perf_counter() - t0

    gpu, power = card()
    for mode, kind in ((pkg.RESIZE_TRAIN, "RandomResizedCrop"), (pkg.RESIZE_EVAL, f"Resize({resize_size}) + CenterCrop")):
        best = None
        for _ in range(rounds):
            r = (timed(calls[mode], iters), timed(plain, iters))
            best = r if best is None else tuple(min(a, b) for a, b in zip(r, best))
        ms, ms_plain = best
        if mode == pkg.RESIZE_TRAIN:
            src = int((box[:, 2] * box[:, 3]).sum()) * C
        else:
            src = N * min(H, -(-H * H_out // Rh)) * min(W, -(-W * W_out // Rw)) * C
        nbytes = src + N * H_out * W_out * C_out * 2
        cpu_s = torchvision_cpu(mode)
        print(json.dumps({"case": f"resized {kind} {name}", "N": N, "us": ms * 1e3, "plain_us": ms_plain * 1e3,
                          "resized_over_plain": ms / ms_plain, "MB": nbytes / 1e6, "hbm_frac": nbytes / (ms * 1e-3) / 1e9 / HBM,
                          "plain_hbm_frac": (N * H_out * W_out * (C + 2 * C_out)) / (ms_plain * 1e-3) / 1e9 / HBM,
                          "torchvision_cpu_ms": cpu_s * 1e3, "torchvision_cpu_over_ours": cpu_s * 1e3 / ms, "vec": info["vec"],
                          "grid": info["grid"], "rows_per_cta": info["rows_per_cta"], "smem": info["smem"], "gpu": gpu,
                          "power_limit": power}), flush=True)


def run_trivial(name, N, H, W, C, C_out, pad, crop, iters, batches=4, row_pitch=0, image_rows=0, rounds=3, erase_p=0.1):
    """one training batch with TrivialAugmentWide (BILINEAR) and RandomErasing(erase_p) (pcnn_augment_trivial_u8_bf16) against the
    same batch without them (pcnn_augment_u8_bf16 with pad, or pcnn_augment_resized_u8_bf16's RandomResizedCrop when crop is set),
    alternated over `rounds` rounds (the best of each kept); and torchvision's per-image CPU path for the two stages alone
    (TrivialAugmentWide on the uint8 crop, then ToTensor + Normalize + RandomErasing, bf16), timed once on one thread.  Bytes: the
    geometry's source bytes, the uint16 workspace written and read, and N h w C_out 2 written."""
    import torchvision.transforms as T
    n = N * batches
    images = torch.randint(0, 256, (n, H, W, C), dtype=torch.uint8, device="cuda")
    labels = torch.randint(0, 10, (n,), dtype=torch.uint8, device="cuda")
    mean, std = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)) if C == 3 else (None, None)
    info, _, _ = pkg.augment_trivial_info(n, H, W, C, 0, N, pkg.TRIVIAL_BILINEAR, erase_p, crop_size=crop, pad=pad, flip=1, C_out=C_out,
                                          row_pitch=row_pitch, image_rows=image_rows)
    h, w = info["h"], info["w"]
    x = torch.empty(N * info["image_rows"] * info["row_pitch"], dtype=torch.int16, device="cuda")
    ws = torch.empty(info["ws_bytes"], dtype=torch.uint8, device="cuda")
    lo = torch.empty(N, dtype=torch.uint8, device="cuda")
    steps = iter(range(1 << 40))
    kw = dict(flip=1, seed=11, epoch=3, mean=mean, std=std, C_out=C_out, row_pitch=row_pitch, image_rows=image_rows)
    first = lambda: (next(steps) % batches) * N
    ours = lambda: eng.augment_trivial(images, labels, n, H, W, C, first(), N, x, ws, lo, trivial=pkg.TRIVIAL_BILINEAR, erase_p=erase_p,
                                       crop_size=crop, pad=pad, **kw)
    if crop is None:
        base = lambda: eng.augment(images, labels, n, H, W, C, first(), N, x, lo, pad=pad, **kw)
    else:
        base = lambda: eng.augment_resized(images, labels, n, H, W, C, first(), N, x, h, w, lo, **kw)
    best = None
    for _ in range(rounds):
        r = (timed(ours, iters), timed(base, iters))
        best = r if best is None else tuple(min(a, b) for a, b in zip(r, best))
    ms, ms_base = best
    src = N * (H * W if crop is None else h * w) * C                  # the RRC box covers at most the image; its mean is near h w
    nbytes = src + 2 * N * h * info["ws_pitch"] * 2 + N * h * w * C_out * 2
    host = torch.randint(0, 256, (N, C, h, w), dtype=torch.uint8)
    ta = T.TrivialAugmentWide(interpolation=T.InterpolationMode.BILINEAR)
    er = T.RandomErasing(p=erase_p, value=0)
    m_t = torch.tensor(mean or (0.0,) * C).view(-1, 1, 1)
    s_t = torch.tensor(std or (1.0,) * C).view(-1, 1, 1)
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    t0 = time.perf_counter()
    for j in range(N):
        er((ta(host[j]).float() / 255.0 - m_t) / s_t).to(torch.bfloat16)
    cpu_s = time.perf_counter() - t0
    torch.set_num_threads(threads)
    gpu, power = card()
    print(json.dumps({"case": f"trivial {name}", "N": N, "us": ms * 1e3, "without_us": ms_base * 1e3, "with_over_without": ms / ms_base,
                      "MB": nbytes / 1e6, "hbm_frac": nbytes / (ms * 1e-3) / 1e9 / HBM, "torchvision_cpu_ms": cpu_s * 1e3,
                      "torchvision_cpu_over_ours": cpu_s * 1e3 / ms, "smem": info["smem"], "grid": info["grid"], "gpu": gpu,
                      "power_limit": power}), flush=True)


def run_resnetgap_resized(iters, rounds=3):
    """one training step of the GAP ResNet at N = 128 fed by pkg.ImageBatcher with crop_size 28 and scale (0.6, 1.0) (shuffle),
    against the same step on the plain batcher (shuffle, pad 2), alternated over `rounds` rounds (the best of each kept)"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from example_nets import ResNetGAP
    g = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    make = lambda **k: pkg.ImageBatcher(eng, g["train_u8"].reshape(-1, 28, 28), g["train_labels"], ResNetGAP.NB, shuffle=True, seed=5,
                                        row_pitch=32, image_rows=28, **k)
    plain_b, res_b = make(pad=2), make(crop_size=28, scale=(0.6, 1.0))
    net = ResNetGAP(eng, pkg, ResNetGAP.init_params())
    k = iter(range(1 << 40))

    def step(batcher):
        net.forward(*batcher.batch(next(k) % batcher.steps_per_epoch))
        net.backward()
        net.sgd(ResNetGAP.LR_STEP)

    gpu, power = card()
    best = None
    for _ in range(rounds):
        r = (timed(lambda: step(res_b), iters), timed(lambda: step(plain_b), iters),
             timed(lambda: res_b.batch(next(k) % res_b.steps_per_epoch), iters))
        best = r if best is None else tuple(min(a, b) for a, b in zip(r, best))
    ms_res, ms_plain, ms_batch = best
    print(json.dumps({"case": f"GAP ResNet training step N={ResNetGAP.NB}, RandomResizedCrop(28) batch vs plain batch (pad 2)",
                      "ms_resized": ms_res, "ms_plain": ms_plain, "resized_over_plain": ms_res / ms_plain, "batch_us": ms_batch * 1e3,
                      "gpu": gpu, "power_limit": power}), flush=True)
    for a in (plain_b, res_b, net):
        a.close()


def run_resnetgap_trivial(iters, rounds=3):
    """one training step of the GAP ResNet at N = 128 fed by pkg.ImageBatcher with pad 2, TrivialAugmentWide (BILINEAR) and
    RandomErasing(0.1) (shuffle), against the same step on the batcher without the two stages, alternated over `rounds` rounds (the
    best of each kept)"""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from example_nets import ResNetGAP
    g = np.load(os.path.join(ROOT, "tests", "golden", "mnist_subset.npz"))
    make = lambda **k: pkg.ImageBatcher(eng, g["train_u8"].reshape(-1, 28, 28), g["train_labels"], ResNetGAP.NB, pad=2, shuffle=True,
                                        seed=5, row_pitch=32, image_rows=28, **k)
    plain_b, ta_b = make(), make(trivial_augment="bilinear", random_erase=0.1)
    net = ResNetGAP(eng, pkg, ResNetGAP.init_params())
    k = iter(range(1 << 40))

    def step(batcher):
        net.forward(*batcher.batch(next(k) % batcher.steps_per_epoch))
        net.backward()
        net.sgd(ResNetGAP.LR_STEP)

    gpu, power = card()
    best = None
    for _ in range(rounds):
        r = (timed(lambda: step(ta_b), iters), timed(lambda: step(plain_b), iters),
             timed(lambda: ta_b.batch(next(k) % ta_b.steps_per_epoch), iters))
        best = r if best is None else tuple(min(a, b) for a, b in zip(r, best))
    ms_ta, ms_plain, ms_batch = best
    print(json.dumps({"case": f"GAP ResNet training step N={ResNetGAP.NB}, pad 2 + TrivialAugmentWide + RandomErasing(0.1) vs pad 2",
                      "ms_trivial": ms_ta, "ms_plain": ms_plain, "trivial_over_plain": ms_ta / ms_plain, "batch_us": ms_batch * 1e3,
                      "gpu": gpu, "power_limit": power}), flush=True)
    for a in (plain_b, ta_b, net):
        a.close()


def run_mbconv(N, iters, hid=16, drop_p=0.0):
    """one training step of an EfficientNet MBConv block with SiLU and squeeze-and-excitation at 28x28x40, N = 128: 1x1 expand to
    240 -> BN + SiLU -> depthwise 5x5 pad 2 -> BN + SiLU -> SE 240 -> hid -> 240 -> 1x1 project to 40 -> BN + x0, its backward (the
    shortcut's gradient dres left apart, as run_mbblock) and the sgd of the eight layers, on the engine's stream.  Next to it the
    torch eager step of the same block on bf16 channels-last tensors (fp32 masters, w -= lr * grad, re-cast to bf16).  With drop_p,
    instead of torch: the same step with stochastic depth (the last BN without r, a DropoutLayer adding x0 to the dropped branch),
    the two steps alternated over three rounds, the best of each kept."""
    H = W = 28
    C, E, k = 40, 240, 5
    r = np.random.default_rng(14)
    u = lambda shape, fan: r.uniform(-1, 1, shape).astype(np.float32) / np.float32(np.sqrt(fan))
    fe, fd, fp = u((E, 1, 1, C), C), u((E, k, k), k * k), u((C, 1, 1, E), E)
    w1, b1_, w2, b2_ = u((hid, E), E), u(hid, E), u((E, hid), hid), u(E, hid)
    ex = pkg.ConvLayer(eng, N, H, W, C, E, 1, 1, fe, None, act=0)
    dwl = pkg.DepthwiseConvLayer(eng, N, H, W, E, k, k, fd, None, act=0, padding=(k // 2, k // 2))
    pr = pkg.ConvLayer(eng, N, H, W, E, C, 1, 1, fp, None, act=0)
    se = pkg.SqueezeExcitationLayer(eng, N, H, W, E, hid, w1, b1_, w2, b2_, act=0)
    b1, b2 = pkg.BatchNormLayer(eng, N, H, W, E, act=pkg.ACT_SILU), pkg.BatchNormLayer(eng, N, H, W, E, act=pkg.ACT_SILU)
    b3 = pkg.BatchNormLayer(eng, N, H, W, C, act=0)
    wide = lambda: torch.empty((N, H, W, E), dtype=torch.int16, device="cuda")
    narrow = lambda: torch.empty((N, H, W, C), dtype=torch.int16, device="cuda")
    x0 = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    dout = torch.randint(0, 0x3F80, (N, H, W, C), dtype=torch.int16, device="cuda")
    dout ^= torch.randint(0, 2, (N, H, W, C), dtype=torch.int16, device="cuda") << 15
    ye, ze, yd, zd, ys, dys, dze, dye, dyd, dzd = (wide() for _ in range(10))
    yp, out, dyp, dres, dx0 = (narrow() for _ in range(5))
    lr = 0.05
    gpu, power = card()
    layers = (ex, b1, dwl, b2, se, pr, b3)

    def step():
        ex.forward(x0, ye); b1.forward(ye, ze); dwl.forward(ze, yd); b2.forward(yd, zd); se.forward(zd, ys); pr.forward(ys, yp)
        b3.forward(yp, out, r=x0)
        b3.backward(out, dout, dyp, dr=dres); pr.backward(yp, dyp, dys); se.backward(ys, dys, dzd); b2.backward(zd, dzd, dyd)
        dwl.backward(yd, dyd, dze); b1.backward(ze, dze, dye); ex.backward(ye, dye, dx0)
        for layer in layers:
            layer.sgd(lr)

    if drop_p:
        dp = pkg.DropoutLayer(eng, N, H * W * C, drop_p, seed=5, per_sample=True)
        bo, dbo = narrow(), narrow()

        def step_drop():
            ex.forward(x0, ye); b1.forward(ye, ze); dwl.forward(ze, yd); b2.forward(yd, zd); se.forward(zd, ys); pr.forward(ys, yp)
            b3.forward(yp, bo); dp.forward(bo, out, r=x0)
            dp.backward(dout, dbo); b3.backward(bo, dbo, dyp); pr.backward(yp, dyp, dys); se.backward(ys, dys, dzd)
            b2.backward(zd, dzd, dyd); dwl.backward(yd, dyd, dze); b1.backward(ze, dze, dye); ex.backward(ye, dye, dx0)
            for layer in layers:
                layer.sgd(lr)

        fused, dropped = float("inf"), float("inf")
        for _ in range(3):
            fused, dropped = min(fused, timed(step, iters)), min(dropped, timed(step_drop, iters))
        ms_dp = {"fwd": timed(lambda: dp.forward(bo, out, r=x0), iters), "bwd": timed(lambda: dp.backward(dout, dbo), iters)}
        print(json.dumps({"case": f"MBConv 28x28x40 -> 240 dw 5x5, SiLU, SE 240 -> {hid} -> 240 training step N={N}, stochastic depth "
                          f"p={drop_p} vs residual fused in BN", "fused_ms": fused, "drop_path_ms": dropped, "extra_ms": dropped - fused,
                          "drop_over_fused": dropped / fused, "drop_fwd_us": ms_dp["fwd"] * 1e3, "drop_bwd_us": ms_dp["bwd"] * 1e3,
                          "gpu": gpu, "power_limit": power}), flush=True)
        for layer in layers:
            layer.close()
        return
    ms = timed(step, iters)
    ms_bn ={"fwd": timed(lambda: b2.forward(yd, zd), iters), "bwd": timed(lambda: b2.backward(zd, dzd, dyd), iters)}
    F = torch.nn.functional
    xt = x0.view(torch.bfloat16).permute(0, 3, 1, 2).detach().requires_grad_(True)
    dt = dout.view(torch.bfloat16).permute(0, 3, 1, 2)
    cl = lambda a: torch.from_numpy(a).to("cuda").contiguous(memory_format=torch.channels_last)
    m32 = {"fe": cl(fe.transpose(0, 3, 1, 2)), "fd": cl(fd[:, None]), "fp": cl(fp.transpose(0, 3, 1, 2))}
    m32.update({kk: torch.from_numpy(v).to("cuda") for kk, v in (("w1", w1), ("v1", b1_), ("w2", w2), ("v2", b2_))})
    for i, ch in ((1, E), (2, E), (3, C)):
        m32[f"g{i}"], m32[f"b{i}"] = torch.ones(ch, device="cuda"), torch.zeros(ch, device="cuda")
    mb = {kk: (v.to(torch.bfloat16) if kk[0] in "fwv" else v.clone()).requires_grad_(True) for kk, v in m32.items()}
    stats = [torch.zeros(ch, device="cuda") if j % 2 == 0 else torch.ones(ch, device="cuda") for ch in (E, E, C) for j in range(2)]

    def torch_step():
        for v in mb.values():
            v.grad = None
        xt.grad = None
        h = F.silu(F.batch_norm(F.conv2d(xt, mb["fe"]), stats[0], stats[1], mb["g1"], mb["b1"], training=True))
        h = F.silu(F.batch_norm(F.conv2d(h, mb["fd"], padding=k // 2, groups=E), stats[2], stats[3], mb["g2"], mb["b2"], training=True))
        s = torch.sigmoid(F.linear(torch.relu(F.linear(h.mean((2, 3)), mb["w1"], mb["v1"])), mb["w2"], mb["v2"]))
        h = h * s[:, :, None, None]
        h = F.batch_norm(F.conv2d(h, mb["fp"]), stats[4], stats[5], mb["g3"], mb["b3"], training=True) + xt
        h.backward(dt)
        with torch.no_grad():
            for kk in m32:
                m32[kk].add_(mb[kk].grad.float(), alpha=-lr)
                mb[kk].copy_(m32[kk])

    ms_torch = timed(torch_step, iters)
    print(json.dumps({"case": f"MBConv 28x28x40 -> 240 dw 5x5, SiLU, SE 240 -> {hid} -> 240 training step N={N}", "ms": ms,
                      "torch_eager_ms": ms_torch, "ours_over_torch": ms / ms_torch, "bn_silu_fwd_ms": ms_bn["fwd"],
                      "bn_silu_bwd_ms": ms_bn["bwd"], "families": [ex.family, pr.family], "gpu": gpu, "power_limit": power}), flush=True)
    for layer in layers:
        layer.close()


if only == "se":                                                       # squeeze-and-excitation passes, torch beside them
    for args in (("56x56x256", 128, 56, 56, 256), ("28x28x512", 128, 28, 28, 512), ("14x14x1024", 128, 14, 14, 1024),
                 ("7x7x2048", 128, 7, 7, 2048), ("112x112x32", 128, 112, 112, 32), ("56x56x144", 128, 56, 56, 144),
                 ("28x28x240", 128, 28, 28, 240), ("7x7x1152", 128, 7, 7, 1152)):
        run_se(*args, 20)
if only == "seblock":                                                  # one step of an SE basic block, torch eager beside it
    run_seblock(128, 20)
if only == "dwconv":                                                   # depthwise convolution passes, torch beside them
    for args in (("112x112x32 3x3/1", 128, 112, 112, 32, 3, 1, 1), ("112x112x96 3x3/2", 128, 112, 112, 96, 3, 2, 1),
                 ("56x56x144 3x3/1", 128, 56, 56, 144, 3, 1, 1), ("56x56x144 3x3/2", 128, 56, 56, 144, 3, 2, 1),
                 ("28x28x192 3x3/1", 128, 28, 28, 192, 3, 1, 1), ("14x14x384 3x3/1", 128, 14, 14, 384, 3, 1, 1),
                 ("7x7x960 3x3/1", 128, 7, 7, 960, 3, 1, 1), ("28x28x240 5x5/1", 128, 28, 28, 240, 5, 1, 2),
                 ("28x28x240 5x5/2", 128, 28, 28, 240, 5, 2, 2), ("56x56x6 3x3/1 (scalar path)", 128, 56, 56, 6, 3, 1, 1)):
        run_dwconv(*args, 20)
if only == "mbblock":                                                  # one step of an inverted-residual block, torch eager beside it
    run_mbblock(128, 20, 3)
    run_mbblock(128, 20, 5)
if only == "gconv":                                                    # grouped convolution passes, torch beside them
    for args in (("resnext 56x56x128 G32 3x3/1", 128, 56, 56, 128, 128, 32, 3, 1, 1),
                 ("resnext 56x56x256->28x28 G32 3x3/2", 128, 56, 56, 256, 256, 32, 3, 2, 1),
                 ("resnext 28x28x256 G32 3x3/1", 128, 28, 28, 256, 256, 32, 3, 1, 1),
                 ("resnext 14x14x512 G32 3x3/1 (Cg 16)", 128, 14, 14, 512, 512, 32, 3, 1, 1),
                 ("resnext 7x7x1024 G32 3x3/1 (Cg 32)", 128, 7, 7, 1024, 1024, 32, 3, 1, 1),
                 ("regnet 28x28x64 G4 3x3/1 (Cg 16)", 128, 28, 28, 64, 64, 4, 3, 1, 1),
                 ("regnet 7x7x384 G24 3x3/1 (Cg 16)", 128, 7, 7, 384, 384, 24, 3, 1, 1),
                 ("multiplier 56x56x32->64 G32 3x3/1", 128, 56, 56, 32, 64, 32, 3, 1, 1),
                 ("shufflenet 28x28x384 G8 1x1", 128, 28, 28, 384, 384, 8, 1, 1, 0)):
        run_gconv(*args, 20)
if only == "resnextblock":                                             # one step of a ResNeXt bottleneck, torch eager beside it
    run_resnextblock(128, 20)
if only == "optim":                                                    # the fused optimizers over the ResNet-18 table, torch beside them
    run_optim(50)
if only == "resnetgap-optim":                                          # the GAP ResNet step with each update, alternated
    run_resnetgap_optim(128, 20)
if only == "avgpool":                                                  # average pooling between layers, torch beside it
    run_avgpool("112x112x64, 2x2/2", 128, 112, 112, 64, 2, 2, 0, 1, 20)
    run_avgpool("56x56x128, 2x2/2", 128, 56, 56, 128, 2, 2, 0, 1, 20)
    run_avgpool("28x28x256, 3x3/1 pad 1, count_include_pad", 128, 28, 28, 256, 3, 1, 1, 1, 20)
    run_avgpool("28x28x256, 3x3/1 pad 1, in-image count", 128, 28, 28, 256, 3, 1, 1, 0, 20)
    run_avgpool("LeNet 24x24x6, 2x2/2 (scalar path)", 1024, 24, 24, 6, 2, 2, 0, 1, 20)
if only == "gap":                                                      # global average pooling, torch beside it
    run_gap("7x7x512", 128, 7, 7, 512, 50)
    run_gap("7x7x2048", 128, 7, 7, 2048, 50)
    run_gap("14x14x256", 128, 14, 14, 256, 50)
    run_gap("56x56x64", 128, 56, 56, 64, 50)
    run_gap("56x56x256 (split path)", 8, 56, 56, 256, 50)
if only == "resnetgap":                                                # one step of the GAP ResNet, torch eager beside it
    run_resnetgap(128, 20)
if only == "bnact":                                                    # BN + ReLU / SiLU / hard-swish / ReLU6, torch beside them
    run_bnact("56x56x64", 128, 56, 56, 64, 50)
    run_bnact("28x28x128", 128, 28, 28, 128, 50)
    run_bnact("14x14x256", 128, 14, 14, 256, 50)
    run_bnact("7x7x256", 128, 7, 7, 256, 50)
    run_bnact("24x24x6 (scalar path)", 1024, 24, 24, 6, 50)
if only == "mbconv":                                                   # one step of an MBConv block with SiLU and SE, torch beside it
    run_mbconv(128, 20)
if only == "dropout":                                                  # dropout and stochastic depth, torch beside them
    for args in (("56x56x64", 128, 56, 56, 64), ("28x28x240", 128, 28, 28, 240), ("7x7x1280", 128, 7, 7, 1280), ("fc 4096", 128, 1, 1, 4096)):
        run_dropout(*args, 50, per_sample=False)
    for args in (("56x56x24", 128, 56, 56, 24), ("28x28x40", 128, 28, 28, 40), ("14x14x112", 128, 14, 14, 112), ("7x7x320", 128, 7, 7, 320)):
        run_dropout(*args, 50, per_sample=True)
if only == "augment":                                                  # the input pipeline, torch eager beside it
    run_augment("28x28x1 -> [28][32]", 1024, 28, 28, 1, 1, 2, 50, row_pitch=32, image_rows=28)
    run_augment("32x32x3 -> 3", 512, 32, 32, 3, 3, 4, 50)
    run_augment("32x32x3 -> 8", 512, 32, 32, 3, 8, 4, 50)
    run_augment("64x64x3 -> 8", 256, 64, 64, 3, 8, 4, 50)
    run_augment("224x224x3 -> 8", 256, 224, 224, 3, 8, 4, 20)
if only == "resnetgap-augment":                                        # the GAP ResNet step fed by the batcher vs the pre-converted slice
    run_resnetgap_augment(20)
if only == "augment-mix":                                              # mixed batches vs the plain batch and torchvision
    run_augment_mix("28x28x1 -> [28][32]", 1024, 28, 28, 1, 1, 2, 50, row_pitch=32, image_rows=28)
    run_augment_mix("32x32x3 -> 3", 512, 32, 32, 3, 3, 4, 50)
    run_augment_mix("32x32x3 -> 8", 512, 32, 32, 3, 8, 4, 50)
    run_augment_mix("64x64x3 -> 8", 256, 64, 64, 3, 8, 4, 50)
    run_augment_mix("224x224x3 -> 8", 256, 224, 224, 3, 8, 4, 20)
if only == "resnetgap-mix":                                            # the GAP ResNet step, mixed + soft loss vs plain + hard loss
    run_resnetgap_mix(20)
if only == "resized":                                                  # resized batches vs the plain batch and torchvision's CPU path
    run_resized("28x28x1 -> 28 [28][32]", 1024, 28, 28, 1, 28, 28, 1, 50, 28, row_pitch=32, image_rows=28)
    run_resized("32x32x3 -> 32, 3", 512, 32, 32, 3, 32, 32, 3, 50, 36)
    run_resized("32x32x3 -> 32, 8", 512, 32, 32, 3, 32, 32, 8, 50, 36)
    run_resized("64x64x3 -> 56, 8", 256, 64, 64, 3, 56, 56, 8, 50, 64)
    run_resized("256x256x3 -> 224, 8", 256, 256, 256, 3, 224, 224, 8, 20, 256)
    run_resized("320x240x3 -> 224, 8", 256, 320, 240, 3, 224, 224, 8, 20, 256)
if only == "trivial":                                                  # TrivialAugmentWide + RandomErasing vs the batch without them
    run_trivial("28x28x1 pad 2 [28][32]", 1024, 28, 28, 1, 1, 2, None, 50, row_pitch=32, image_rows=28)
    run_trivial("32x32x3 pad 4, 3", 512, 32, 32, 3, 3, 4, None, 50)
    run_trivial("256x256x3 -> 224 RRC, 8", 256, 256, 256, 3, 8, 0, (224, 224), 20)
if only == "resnetgap-trivial":                                        # the GAP ResNet step, with and without the two stages
    run_resnetgap_trivial(20)
if only == "resnetgap-resized":                                        # the GAP ResNet step, resized batch vs plain batch
    run_resnetgap_resized(20)
if only == "mbconvdrop":                                               # the MBConv step with stochastic depth against the fused residual
    run_mbconv(128, 20, drop_p=0.2)
if only == "bn":                                                       # batch normalization passes, torch beside them
    run_bn("56x56x64", 128, 56, 56, 64, 50)
    run_bn("28x28x128", 128, 28, 28, 128, 50)
    run_bn("14x14x256", 128, 14, 14, 256, 50)
    run_bn("7x7x256", 128, 7, 7, 256, 50)
    run_bn("24x24x6 (scalar path)", 1024, 24, 24, 6, 50)
if only == "resblock":                                                 # one step of a ResNet basic block, torch eager beside it
    run_resblock(128, 20)
if only == "linear":                                                   # fully connected passes, torch.nn.functional.linear beside them
    run_linear("7x7x256 -> 256", 1024, 7, 7, 256, 256, 0, 50)
    run_linear("1x1x2048 -> 256", 4096, 1, 1, 2048, 256, 0, 50)
    run_linear("6x6x16 -> 128 sigmoid (fc1)", 1024, 6, 6, 16, 128, 1, 50)
    run_linear("128 -> 10 (fc2)", 1024, 1, 1, 128, 10, 0, 50)
if only == "classifier":                                               # one step of the LeNet-style classifier, torch eager beside it
    run_classifier(1024, 50)
    run_classifier(1024, 50, relu=True)
if only == "pool":                                                     # max pooling between conv layers, torch beside it
    run_pool("LeNet c1 output 24x24x6, 2x2/2", 1024, 24, 24, 6, 2, 2, 0, 20)
    run_pool("112x112x64, 2x2/2", 128, 112, 112, 64, 2, 2, 0, 20)
    run_pool("112x112x64, 3x3/2 pad 1", 128, 112, 112, 64, 3, 2, 1, 20)
    run_pool("56x56x128, 2x2/2", 128, 56, 56, 128, 2, 2, 0, 20)
    run_pool("28x28x256, 2x2/2", 128, 28, 28, 256, 2, 2, 0, 20)
if only == "train":                                                    # a ConvLayer training step, pass by pass, and torch eager
    run_train("56x56x64->64 3x3 pad 1", 128, 56, 56, 64, 64, 3, 3, 1, 1, 20)
    run_train("28x28x128->128 3x3 pad 1", 128, 28, 28, 128, 128, 3, 3, 1, 1, 20)
    run_train("14x14x256->256 3x3 pad 1", 128, 14, 14, 256, 256, 3, 3, 1, 1, 20)
    run_train("56x56x64->128 3x3 stride 2 pad 1", 128, 56, 56, 64, 128, 3, 3, 2, 1, 20)
    run_train("LeNet c1 28x28x1->6 5x5", 1024, 28, 28, 1, 6, 5, 5, 1, 0, 20, with_dx=False)
    run_train("56x56x64->64 3x3 pad 1", 128, 56, 56, 64, 64, 3, 3, 1, 1, 20, act=3)            # the same layers with ReLU
    run_train("28x28x128->128 3x3 pad 1", 128, 28, 28, 128, 128, 3, 3, 1, 1, 20, act=3)
    run_train("14x14x256->256 3x3 pad 1", 128, 14, 14, 256, 256, 3, 3, 1, 1, 20, act=3)
    run_train("56x56x64->128 3x3 stride 2 pad 1", 128, 56, 56, 64, 128, 3, 3, 2, 1, 20, act=3)
    run_train("LeNet c1 28x28x1->6 5x5", 1024, 28, 28, 1, 6, 5, 5, 1, 0, 20, with_dx=False, act=3)
if only == "widesame":                                                 # "same" layers: built-in padding, pad-copy route, cuDNN
    run_wide_same("56x56x64->64 3x3 pad 1", 128, 56, 56, 64, 64, 3, 3, 1, 1, 20)
    run_wide_same("28x28x128->128 3x3 pad 1", 128, 28, 28, 128, 128, 3, 3, 1, 1, 20)
    run_wide_same("14x14x256->256 3x3 pad 1", 128, 14, 14, 256, 256, 3, 3, 1, 1, 20)
    run_wide_same("56x56x64->128 3x3 stride 2 pad 1", 128, 56, 56, 64, 128, 3, 3, 2, 1, 20)
if only == "wide":                                                     # wide channel counts (WideConvPlan), cuDNN beside them
    run_wide("56x56x64->64 3x3", 128, 56, 56, 64, 64, 3, 3, 1, 20)
    run_wide("28x28x128->128 3x3", 128, 28, 28, 128, 128, 3, 3, 1, 20)
    run_wide("14x14x256->256 3x3", 128, 14, 14, 256, 256, 3, 3, 1, 20)
    run_wide("56x56x64->256 1x1", 128, 56, 56, 64, 256, 1, 1, 1, 20)
    run_wide("56x56x64->128 3x3 stride 2", 128, 56, 56, 64, 128, 3, 3, 2, 20)
if only == "widebwd":                                                  # gradients of the same five layers, cuDNN beside them
    run_wide_bwd("56x56x64->64 3x3", 128, 56, 56, 64, 64, 3, 3, 1, 20)
    run_wide_bwd("28x28x128->128 3x3", 128, 28, 28, 128, 128, 3, 3, 1, 20)
    run_wide_bwd("14x14x256->256 3x3", 128, 14, 14, 256, 256, 3, 3, 1, 20)
    run_wide_bwd("56x56x64->256 1x1", 128, 56, 56, 64, 256, 1, 1, 1, 20)
    run_wide_bwd("56x56x64->128 3x3 stride 2", 128, 56, 56, 64, 128, 3, 3, 2, 20)
if only in ("all", "bwd"):
    for N in (8, 32, 128):
        run_bwd("224x224x3->64x3x3 bf16 (config 5)", N, 224, 224, 3, 64, 3, 3, 10)
if only == "bwdpad":                                                   # filter counts padded to 64: 32 filters, and LeNet's own 6
    run_bwd("224x224x3->32x3x3 bf16 (padded to 64 filters)", 128, 224, 224, 3, 32, 3, 3, 10)
    run_bwd("224x224x3->16x3x3 bf16 (padded to 64 filters)", 128, 224, 224, 3, 16, 3, 3, 10)
if only == "bwdk128":                                                  # 128 filters: two 64-filter groups per dy row
    run_bwd("224x224x3->128x3x3 bf16", 64, 224, 224, 3, 128, 3, 3, 10)
if only == "bwd128":                                                   # the profiler's target: few launches
    run_bwd("224x224x3->64x3x3 bf16 (config 5)", 128, 224, 224, 3, 64, 3, 3, 2)
if only == "bwds2":                                                    # config 5 at stride 2 next to stride 1 (same launch count)
    run_bwd("224x224x3->64x3x3 bf16 (config 5)", 128, 224, 224, 3, 64, 3, 3, 10)
    run_bwd("224x224x3->64x3x3 bf16 (config 5), stride 2", 128, 224, 224, 3, 64, 3, 3, 10, stride=2)
if only in ("all", "lenet"):
    for N in (1024, 8192, 65536):
        run("lenet_c1_bf16_sigmoid (config 3 shape)", N, 28, 28, 1, 6, 5, 5, 1, 20)
    for N in (8192, 65536):
        run("lenet_c1_bf16_sigmoid, 32-row image pitch (rows 28..31 padding)", N, 28, 28, 1, 6, 5, 5, 1, 20, image_rows=32)
if only == "lenet1024":                                                # BASELINE configs[2]: LeNet c1 shape, batch 1024
    run("lenet_c1_bf16_sigmoid (config 3 shape)", 1024, 28, 28, 1, 6, 5, 5, 1, 2)
if only == "fwd128":                                                   # the profiler's target
    run("224x224x3->64x3x3 bf16 (config 5)", 128, 224, 224, 3, 64, 3, 3, 0, 2)
if only == "stprobe":                                                  # the store phase of the forward epilogue alone
    N, P, H, RE = 128, 222, 224, 222 * 64
    y = torch.empty((N, P, RE), dtype=torch.int16, device="cuda")
    for mode in (0, 2, 5, 6):
        for hot in (0, 1):
            g = eng.measure_tma_write(y, N, P, H, RE, mode, hot, 10)
            print(json.dumps({"case": "tma store probe", "mode": mode, "hot_l2_target": hot, "GBps": g, "us_per_launch": N * P * RE * 2 / g / 1e3}), flush=True)
if only == "fwdq":                                                     # one line: forward at N = 128 without bias
    run("224x224x3->64x3x3 bf16 (config 5), no bias", 128, 224, 224, 3, 64, 3, 3, 0, 20, bias=False)
if only == "fwdab":                                                    # forward at N = 128: with / without bias, with sigmoid
    run("224x224x3->64x3x3 bf16 (config 5), bias", 128, 224, 224, 3, 64, 3, 3, 0, 20)
    run("224x224x3->64x3x3 bf16 (config 5), no bias", 128, 224, 224, 3, 64, 3, 3, 0, 20, bias=False)
    run("224x224x3->64x3x3 bf16 (config 5), bias + sigmoid", 128, 224, 224, 3, 64, 3, 3, 1, 20)
    run("lenet_c1_bf16_sigmoid, 32-row image pitch (rows 28..31 padding)", 65536, 28, 28, 1, 6, 5, 5, 1, 20, image_rows=32)
    run("lenet_c1_bf16_sigmoid (config 3 shape)", 65536, 28, 28, 1, 6, 5, 5, 1, 20)
if only in ("all", "cfg5"):
    for N in (1, 8, 32, 128):
        run("224x224x3->64x3x3 bf16 (config 5)", N, 224, 224, 3, 64, 3, 3, 0, 10)
if only == "convt":                                                   # transposed convolutions of an FCN / DCGAN decoder, N = 128
    run_convt("7x7x256->128 4x4/2 pad 1", 128, 7, 7, 256, 128, 4, 2, 1, 20)
    run_convt("14x14x128->64 4x4/2 pad 1", 128, 14, 14, 128, 64, 4, 2, 1, 20)
    run_convt("28x28x64->32 4x4/2 pad 1", 128, 28, 28, 64, 32, 4, 2, 1, 20)
if only == "upsample":                                                 # bilinear x2 / x4 / x8
    run_upsample("28x28x64", 128, 28, 28, 64, 2, 20)
    run_upsample("28x28x21", 64, 28, 28, 21, 4, 20)
    run_upsample("28x28x21", 32, 28, 28, 21, 8, 20)
if only == "segce":                                                    # VOC-sized per-pixel loss
    run_segce(16, 21, 20)
if only == "fcn":
    run_fcn(20)
if only == "dilated":                                                  # dilated wide passes vs cuDNN and vs dilation 1
    for d in (1, 2):
        run_dilated("56x56x64->64 3x3", 128, 56, 56, 64, 64, 3, d, 20)
    for d in (1, 2, 4):
        run_dilated("28x28x128->128 3x3", 256, 28, 28, 128, 128, 3, d, 20)
    for d in (6, 12, 18):                                              # ASPP; N 96 gives every pass more than 2 x stages tiles per CTA
        run_dilated("ASPP 33x33x512->256 3x3", 96, 33, 33, 512, 256, 3, d, 20)
if only == "dwdilated":                                                # dilated depthwise passes vs torch and vs dilation 1
    for d in (1, 2):
        run_dwdilated("56x56x144 3x3", 128, 56, 56, 144, 3, d, 20)
        run_dwdilated("28x28x240 5x5", 128, 28, 28, 240, 5, d, 20)
if only == "deeplab":
    run_deeplab(20)
if only == "gn":                                                       # group normalization passes, torch beside them
    run_gn("56x56x64 G32 (the bn shape)", 128, 56, 56, 64, 32, 20)
    run_gn("128x128x64 G32", 8, 128, 128, 64, 32, 20)
    run_gn("256x256x32 G8, small batch", 2, 256, 256, 32, 8, 20)
    run_gn("28x28x256 G256 (instance norm)", 16, 28, 28, 256, 256, 20)
if only == "nlblock":                                                  # one non-local block training step, torch eager beside it
    run_nlblock("non-local block N128 12x12x16 h1 d16 (NonLocalResNet)", 128, 12, 12, 16, 1, 16, 50)
    run_nlblock("non-local block N128 28x28x64 h1 d64", 128, 28, 28, 64, 1, 64, 20)
if only == "attn":                                                     # self-attention, torch's flash SDPA beside it
    run_attn("BoTNet 14x14 N128 T196 h4 d64", 128, 196, 4, 64, 20)
    run_attn("non-local Res3 N32 T784 h1 d128", 32, 784, 1, 128, 20)
    run_attn("N16 T3136 h1 d64", 16, 3136, 1, 64, 10)
    run_attn("DANet N8 T4096 h1 d64", 8, 4096, 1, 64, 10)
if only == "pixelshuffle":                                             # sub-pixel upsamplers and their inverses, torch beside them
    run_pixelshuffle("128x128x12 -> 256x256x3", 16, 128, 128, 3, 2, 20)
    run_pixelshuffle("64x64x48 -> 256x256x3", 16, 64, 64, 3, 4, 20)
    run_pixelshuffle("EDSR 48x48x256 -> 96x96x64", 16, 48, 48, 64, 2, 20)
    run_pixelshuffle("EDSR 96x96x256 -> 192x192x64", 16, 96, 96, 64, 2, 20)
    run_pixelshuffle("28x28x256 -> 56x56x64", 128, 28, 28, 64, 2, 20)
if only == "regloss":                                                  # MSE and L1 with their gradients, torch beside them
    run_regloss("16x256x256x3", 16, 256, 256, 3, 20)
    run_regloss("16x192x192x64", 16, 192, 192, 64, 20)
if only == "latent":                                                   # the VAE latent: a dense head, a spatial latent, a wide one
    for name, R, L in (("fc 65536x128", 65536, 128), ("spatial 16x256x256x4", 16 * 256 * 256, 4), ("fc 8192x1024", 8192, 1024)):
        run_latent(name, R, L, 20)
if only == "bce":                                                      # ConvVAE's head, a segmentation head, a multi-label head
    run_bce("128x784x1 ts8", 128 * 784, 1, 8, 20)
    run_bce("16x256x256x8", 16 * 256 * 256, 8, 8, 20)
    run_bce("65536x80", 65536, 80, 80, 20)
if only == "vae":
    run_vae(20)
if only == "espcn":
    run_restorer("ESPCNLite", 20)
if only == "denoise":
    run_restorer("DenoiseNet", 20)
eng.close()
if only == "wprobe":                                                   # what a pure WRITE stream / pure READ stream / copy reach on this GPU
    # library fill / reduce / copy kernels as a yardstick for the store-dominated forward pass (807 MB written, 39 MB read):
    # the data-sheet HBM number counts reads and writes together
    nbytes = 807 << 20
    buf = torch.empty((nbytes // 4,), dtype=torch.int32, device="cuda")
    src = torch.ones((nbytes // 4,), dtype=torch.int32, device="cuda")
    def timeit(fn, iters=20):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(iters):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters
    ms_fill = timeit(lambda: buf.fill_(7))
    ms_memset = timeit(lambda: buf.zero_())
    ms_copy = timeit(lambda: buf.copy_(src))
    ms_read = timeit(lambda: src.sum())
    print(json.dumps({"case": "write/read/copy yardsticks (torch library kernels, 807 MiB)", "fill_GBps": nbytes / ms_fill / 1e6,
                      "memset_GBps": nbytes / ms_memset / 1e6, "copy_GBps_read_plus_write": 2 * nbytes / ms_copy / 1e6,
                      "reduce_read_GBps": nbytes / ms_read / 1e6, "hbm_peak_file": HBM}), flush=True)
