"""GPU parity tests of the bf16 wgmma convolution (csrc/conv_tc.cu, SURVEY.md x3).

PARITY UNPINNED by the reference (no bf16 / tensor-core path exists there).  The checker is the direct convolution
orc_conv_fwd_nhwc (oracle/lenet_oracle.c: the reference's conv semantics, layer.h:118-130, generalised to C channels and
K filters, double accumulation) evaluated on the SAME bf16-rounded activations and filters, so the only differences are
fp32 accumulation order in the tensor core and the final bf16 rounding of the output:
    |d| <= 2^-8 |ref| + 1e-3   per element,   rel-L2 <= 4e-3     (stated bound of SURVEY.md 8c item 5: 2e-2)
"""
import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu


def conv_case(eng, pkg, N, H, W, C, K, R, S, act, seed, real=None, stride=1):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0, 1, (N, H, W, C)).astype(np.float32) if real is None else real        # config 5: x ~ U[0,1)
    f = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)                                # same law as layer.h:49-52
    b = rng.uniform(-0.5, 0.5, K).astype(np.float32)
    xb = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(x))
    fb = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(f))
    P, Q = (H - R) // stride + 1, (W - S) // stride + 1
    ref = np.empty((N, P, Q, K), np.float32)
    O.oracle().orc_conv_fwd_nhwc_strided(O.fp(xb.reshape(-1)), O.fp(fb.reshape(-1)), O.fp(b), O.fp(ref.reshape(-1)), N, H, W, C, K, R, S, stride)
    if stride == 1:          # the strided restatement at stride 1 IS the stride-1 oracle
        ref1 = np.empty_like(ref)
        O.oracle().orc_conv_fwd_nhwc(O.fp(xb.reshape(-1)), O.fp(fb.reshape(-1)), O.fp(b), O.fp(ref1.reshape(-1)), N, H, W, C, K, R, S)
        assert np.array_equal(ref, ref1)
    if act:
        ref = (1.0 / (1.0 + np.exp(-ref.astype(np.float64)))).astype(np.float32)
    pitch = (W * C + 7) // 8 * 8
    xp = np.zeros((N * H, pitch), np.uint16)
    xp[:, : W * C] = pkg.f32_to_bf16_bits(x).reshape(N * H, W * C)
    plan = pkg.ConvPlan(eng, N, H, W, C, K, R, S, fb, b, act=act, row_pitch=pitch, stride=stride)
    dx = eng.to_device(xp)
    dy = eng.array((N, P, Q, K), np.uint16)
    plan.fwd(dx, dy)
    eng.sync()
    got = pkg.bf16_bits_to_f32(dy.to_host())
    plan.close()
    err = np.abs(got - ref)
    assert np.all(err <= 2.0 ** -8 * np.abs(ref) + 1e-3), (float(err.max()), np.unravel_index(err.argmax(), err.shape))
    rel = np.linalg.norm((got - ref).astype(np.float64)) / np.linalg.norm(ref.astype(np.float64))
    assert rel <= 4e-3, rel
    return rel


def test_lenet_c1_shape_random(eng, pkg):
    # config 3 shape: 28x28x1 -> 6 filters 5x5, 128 images (4 full row-tiles of 128 rows = 28 tiles)
    conv_case(eng, pkg, 128, 28, 28, 1, 6, 5, 5, act=0, seed=1)


def test_lenet_c1_real_digits_with_sigmoid_epilogue(eng, pkg, golden):
    # the c1 layer of the reference on real MNIST digits with the seed-1 filters, bias + sigmoid fused: compare with
    # the fp32 oracle's c1.output (layer.h:105-140 + :85-89) at bf16 resolution
    N = 64
    imgs = O.u8_to_f32(golden["train_u8"][:N]).reshape(N, 28, 28, 1)
    p = golden["params_init"]
    filt = p[0:150].reshape(6, 5, 5, 1)
    bias = p[150:156]
    pitch = 32
    xp = np.zeros((N * 28, pitch), np.uint16)
    xp[:, :28] = pkg.f32_to_bf16_bits(imgs).reshape(N * 28, 28)
    plan = pkg.ConvPlan(eng, N, 28, 28, 1, 6, 5, 5, filt, bias, act=1, row_pitch=pitch)
    dy = eng.array((N, 24, 24, 6), np.uint16)
    plan.fwd(eng.to_device(xp), dy)
    eng.sync()
    got = pkg.bf16_bits_to_f32(dy.to_host())                       # NHWC
    plan.close()
    ref = np.stack([O.forward(p, imgs[s].reshape(-1))[3456:6912].reshape(6, 24, 24) for s in range(N)])   # NCHW fp32
    ref = ref.transpose(0, 2, 3, 1)
    # bf16 inputs/filters (2^-9 relative each) through a 25-term sum and a sigmoid: 2e-2 rel-L2 is SURVEY.md's stated bound
    rel = np.linalg.norm((got - ref).astype(np.float64)) / np.linalg.norm(ref.astype(np.float64))
    assert rel <= 2e-2, rel
    assert np.abs(got - ref).max() <= 3e-2


def test_lenet_c1_with_32_row_image_pitch_uses_tma_stores(eng, pkg, golden):
    # images laid out [N][32 rows][32 cols] (rows 28..31 zero): the 32-row groups of the M dimension coincide with
    # images, so the epilogue takes the asynchronous TMA-store path; output rows p >= 24 are clipped by the tensor map
    N = 96
    imgs = O.u8_to_f32(golden["train_u8"][:N]).reshape(N, 28, 28)
    p = golden["params_init"]
    filt, bias = p[0:150].reshape(6, 5, 5, 1), p[150:156]
    xp = np.zeros((N, 32, 32), np.uint16)
    xp[:, :28, :28] = pkg.f32_to_bf16_bits(imgs)
    plan = pkg.ConvPlan(eng, N, 28, 28, 1, 6, 5, 5, filt, bias, act=0, row_pitch=32, image_rows=32)
    dy = eng.to_device(np.full((N, 24, 24, 6), 0x7FC0, np.uint16))       # NaN canary: every element must be written
    plan.fwd(eng.to_device(xp.reshape(N * 32, 32)), dy)
    eng.sync()
    got = pkg.bf16_bits_to_f32(dy.to_host())
    plan.close()
    xb = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(imgs)).reshape(N, 28, 28, 1)
    fb = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(filt))
    ref = np.empty((N, 24, 24, 6), np.float32)
    O.oracle().orc_conv_fwd_nhwc(O.fp(xb.reshape(-1)), O.fp(fb.reshape(-1)), O.fp(np.ascontiguousarray(bias)), O.fp(ref.reshape(-1)),
                                 N, 28, 28, 1, 6, 5, 5)
    assert np.isfinite(got).all()
    assert np.all(np.abs(got - ref) <= 2.0 ** -8 * np.abs(ref) + 1e-3)


@pytest.mark.parametrize("N,H,W", [(1, 224, 224), (2, 64, 40), (3, 19, 23)])
def test_config5_shape(eng, pkg, N, H, W):
    # 3 input channels, 64 filters of 3x3: pixel blocks of 4, ragged last block (222 = 55 * 4 + 2), ragged row tiles
    conv_case(eng, pkg, N, H, W, 3, 64, 3, 3, act=0, seed=N * 100 + H)


def test_other_small_channel_shapes(eng, pkg):
    conv_case(eng, pkg, 5, 12, 30, 2, 16, 3, 5, act=0, seed=9)      # C = 2, K = 16, 3x5 taps
    conv_case(eng, pkg, 2, 33, 33, 4, 32, 5, 3, act=1, seed=10)     # C = 4, K = 32, 5x3 taps, sigmoid epilogue
    conv_case(eng, pkg, 16, 12, 12, 4, 16, 5, 5, act=1, seed=12)    # C = 4, K = 16, 5x5 taps (20 + alignment remainder <= 32)


@pytest.mark.parametrize("shape", [(3, 28, 28, 1, 16, 5, 5, 2),      # LeNet-sized input, stride 2: 12 x 12 outputs
                                   (2, 64, 40, 3, 64, 3, 3, 2),      # config-5-like layer at stride 2 (ragged pixel blocks)
                                   (1, 224, 224, 3, 64, 3, 3, 2),    # config 5 at stride 2
                                   (2, 33, 30, 2, 32, 3, 3, 3)])     # stride 3, rows per image padded to a multiple of 3
def test_strided_convolution(eng, pkg, shape):
    """SURVEY.md 8f row 4: window step > 1 in the forward plan (the reference's conv is stride 1, layer.h:118-130), against
    orc_conv_fwd_nhwc_strided on the bf16-rounded operands."""
    N, H, W, C, K, R, S, stride = shape
    if H % stride:                       # rows per image must be a multiple of the stride: pad the image with zero rows
        Hp = (H + stride - 1) // stride * stride
        rng = np.random.default_rng(1)
        x = np.zeros((N, Hp, W, C), np.float32)
        x[:, :H] = rng.uniform(0, 1, (N, H, W, C)).astype(np.float32)
        f = rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)
        xb, fb = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(x)), pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(f))
        P, Q = (H - R) // stride + 1, (W - S) // stride + 1
        ref = np.empty((N, P, Q, K), np.float32)
        O.oracle().orc_conv_fwd_nhwc_strided(O.fp(np.ascontiguousarray(xb[:, :H]).reshape(-1)), O.fp(fb.reshape(-1)), O.fp(np.zeros(K, np.float32)),
                                             O.fp(ref.reshape(-1)), N, H, W, C, K, R, S, stride)
        pitch = (W * C + 7) // 8 * 8
        xp = np.zeros((N * Hp, pitch), np.uint16)
        xp[:, : W * C] = pkg.f32_to_bf16_bits(x).reshape(N * Hp, W * C)
        plan = pkg.ConvPlan(eng, N, H, W, C, K, R, S, fb, None, act=0, row_pitch=pitch, image_rows=Hp, stride=stride)
        dy = eng.array((N, P, Q, K), np.uint16)
        plan.fwd(eng.to_device(xp), dy)
        got = pkg.bf16_bits_to_f32(dy.to_host())
        plan.close()
        assert np.all(np.abs(got - ref) <= 2.0 ** -8 * np.abs(ref) + 1e-3)
    else:
        conv_case(eng, pkg, N, H, W, C, K, R, S, act=0, seed=sum(shape), stride=stride)


def test_plan_rejects_unsupported_shapes(eng, pkg):
    with pytest.raises(pkg.PcnnError):
        # the second convolution of the LeNet-5-style variant (12x12x6 -> 16 x 5x5): 5 taps x 6 channels + the 16-byte
        # alignment remainder exceed the 32-element chunk of one filter row -- that layer runs in csrc/lenet5_kernels.cu
        pkg.ConvPlan(eng, 4, 12, 12, 6, 16, 5, 5, np.zeros(16 * 25 * 6, np.float32))
    with pytest.raises(pkg.PcnnError):
        pkg.ConvPlan(eng, 1, 32, 32, 64, 64, 3, 3, np.zeros(64 * 9 * 64, np.float32))      # (Qt+S-1)*C > 32 for every Qt
    with pytest.raises(pkg.PcnnError):
        pkg.ConvPlan(eng, 1, 28, 28, 1, 6, 5, 5, np.zeros(150, np.float32), row_pitch=28)   # pitch not a multiple of 8


@pytest.mark.parametrize("shape", [(4, 28, 28, 1, 6, 5, 5), (2, 40, 36, 3, 64, 3, 3), (3, 17, 21, 2, 16, 3, 5)])
def test_conv_wgrad_and_dgrad_vs_oracle(eng, pkg, shape):
    """Backward passes of the generic convolution (csrc/conv_bwd.cu) against orc_conv_wgrad_nhwc / orc_conv_dgrad_nhwc on
    the same bf16-rounded operands: fp32 accumulation on both sides (the oracle in double), so
    wgrad (fp32 out) rel-L2 <= 1e-5, dgrad (bf16 out) |d| <= 2^-8 |ref| + 1e-3."""
    N, H, W, C, K, R, S = shape
    rng = np.random.default_rng(sum(shape))
    P, Q = H - R + 1, W - S + 1
    x = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(0, 1, (N, H, W, C)).astype(np.float32)))
    dy = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-1, 1, (N, P, Q, K)).astype(np.float32)))     # config 5: dy ~ U[-1,1)
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    dw_ref = np.empty((K, R, S, C), np.float32)
    dx_ref = np.empty((N, H, W, C), np.float32)
    O.oracle().orc_conv_wgrad_nhwc(O.fp(x.reshape(-1)), O.fp(dy.reshape(-1)), O.fp(dw_ref.reshape(-1)), N, H, W, C, K, R, S)
    O.oracle().orc_conv_dgrad_nhwc(O.fp(dy.reshape(-1)), O.fp(f.reshape(-1)), O.fp(dx_ref.reshape(-1)), N, H, W, C, K, R, S)
    dxb, dyb = eng.to_device(pkg.f32_to_bf16_bits(x)), eng.to_device(pkg.f32_to_bf16_bits(dy))
    dw = eng.array((K, R, S, C))
    dxo = eng.array((N, H, W, C), np.uint16)
    # default path = tensor cores only (filter counts that are not a multiple of 64 are zero-padded up to one): a shape they
    # cannot take is an ERROR naming the explicit switch, never a silent detour to the slow kernels
    for op in ("wgrad", "dgrad"):
        try:
            if op == "wgrad":
                eng.conv_wgrad(dxb, dyb, dw, N, H, W, C, K, R, S)
                assert np.linalg.norm((dw.to_host() - dw_ref).astype(np.float64)) / np.linalg.norm(dw_ref.astype(np.float64)) <= 1e-5
            else:
                eng.conv_dgrad(dyb, eng.to_device(f), dxo, N, H, W, C, K, R, S)
                assert np.all(np.abs(pkg.bf16_bits_to_f32(dxo.to_host()) - dx_ref) <= 2.0 ** -8 * np.abs(dx_ref) + 1e-3)
        except pkg.PcnnError as exc:
            assert "pcnn_conv_bwd_select" in str(exc)
    eng.conv_bwd_select(reference=True)                     # the FMA-pipe reference kernels take every shape
    try:
        eng.conv_wgrad(dxb, dyb, dw, N, H, W, C, K, R, S)
        got_w = dw.to_host()
        assert np.linalg.norm((got_w - dw_ref).astype(np.float64)) / np.linalg.norm(dw_ref.astype(np.float64)) <= 1e-5
        eng.conv_wgrad(dxb, dyb, dw, N, H, W, C, K, R, S)
        assert np.array_equal(dw.to_host().view(np.uint32), got_w.view(np.uint32))                              # deterministic
        eng.conv_dgrad(dyb, eng.to_device(f), dxo, N, H, W, C, K, R, S)
        got_x = pkg.bf16_bits_to_f32(dxo.to_host())
        assert np.all(np.abs(got_x - dx_ref) <= 2.0 ** -8 * np.abs(dx_ref) + 1e-3)
    finally:
        eng.conv_bwd_select(reference=False)


@pytest.mark.parametrize("shape", [(8, 28, 28, 1, 6, 5, 5, 32),       # LeNet c1 (6 filters; layer.h:371-395), rows padded to 32 elements
                                   (2, 40, 40, 3, 16, 3, 3, 0),       # 16 filters
                                   (1, 24, 32, 3, 96, 3, 3, 0)])      # 96 filters -> two groups of 64
def test_filter_counts_that_are_not_multiples_of_64_run_on_the_tensor_cores(eng, pkg, shape):
    """K % 64 != 0: dy is zero-padded to the next multiple of 64 filters and the 64-filter wgmma kernels run (VERDICT r1 item 7);
    results against the oracle and against the reference kernels, launch counts prove the tensor-core path ran."""
    N, H, W, C, K, R, S, pitch = shape
    pitch = pitch or W * C
    rng = np.random.default_rng(sum(shape))
    P, Q = H - R + 1, W - S + 1
    x = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(0, 1, (N, H, W, C)).astype(np.float32)))
    dy = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-1, 1, (N, P, Q, K)).astype(np.float32)))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    dw_ref = np.empty((K, R, S, C), np.float32)
    dx_ref = np.empty((N, H, W, C), np.float32)
    O.oracle().orc_conv_wgrad_nhwc(O.fp(x.reshape(-1)), O.fp(dy.reshape(-1)), O.fp(dw_ref.reshape(-1)), N, H, W, C, K, R, S)
    O.oracle().orc_conv_dgrad_nhwc(O.fp(dy.reshape(-1)), O.fp(f.reshape(-1)), O.fp(dx_ref.reshape(-1)), N, H, W, C, K, R, S)
    xp = np.zeros((N, H, pitch), np.uint16)
    xp[:, :, : W * C] = pkg.f32_to_bf16_bits(x).reshape(N, H, W * C)
    dxb, dyb, fd = eng.to_device(xp), eng.to_device(pkg.f32_to_bf16_bits(dy)), eng.to_device(f)
    out = {}
    try:
        for path in ("tc", "fma"):
            eng.conv_bwd_select(reference=(path == "fma"))
            l0 = eng.launch_count()
            dw = eng.array((K, R, S, C))
            eng.conv_wgrad(dxb, dyb, dw, N, H, W, C, K, R, S, row_pitch=pitch)
            got_w = dw.to_host()
            assert np.linalg.norm((got_w - dw_ref).astype(np.float64)) / np.linalg.norm(dw_ref.astype(np.float64)) <= 1e-5, path
            dxo = eng.to_device(np.full((N, H, pitch), 0x4242, np.uint16))
            eng.conv_dgrad(dyb, fd, dxo, N, H, W, C, K, R, S, row_pitch=pitch)
            got_x = pkg.bf16_bits_to_f32(dxo.to_host().reshape(N, H, pitch)[:, :, : W * C].reshape(N, H, W, C))
            assert np.all(np.abs(got_x - dx_ref) <= 2.0 ** -8 * np.abs(dx_ref) + 1e-3), path
            out[path] = eng.launch_count() - l0
    finally:
        eng.conv_bwd_select(reference=False)
    assert out["tc"] != out["fma"]              # different kernels ran (the padded path adds its pad kernels)


def test_lenet_wgrad_matches_reference_bp_weight_c1(eng, pkg, golden):
    """bp_weight_c1 of the reference (layer.h:371-395) = this wgrad / 576 for one sample, up to bf16 rounding of the inputs."""
    p = golden["params_init"]
    img = O.u8_to_f32(golden["train_u8"][0])
    a = O.forward(p, img)
    b = O.backward(p, img, int(golden["train_labels"][0]), a)
    dpre = b[slice(*O.BACK_OFF["c1_dpre"])].reshape(6, 24, 24).transpose(1, 2, 0)           # -> [P][Q][K]
    dw_ref = b[slice(*O.BACK_OFF["g"])][0:150].reshape(6, 5, 5, 1)
    dw = eng.array((6, 5, 5, 1))
    eng.conv_bwd_select(reference=True)                     # 6 filters: no tensor-core kernel
    try:
        eng.conv_wgrad(eng.to_device(pkg.f32_to_bf16_bits(img.reshape(1, 28, 28, 1))), eng.to_device(pkg.f32_to_bf16_bits(dpre)), dw,
                       1, 28, 28, 1, 6, 5, 5)
    finally:
        eng.conv_bwd_select(reference=False)
    got = dw.to_host() / 576.0
    assert np.linalg.norm(got - dw_ref) / np.linalg.norm(dw_ref) <= 1e-2                                       # bf16 operands


BWD_TC_SHAPES = [(1, 224, 224, 3, 64, 3, 3),      # config 5
                 (2, 40, 40, 3, 64, 3, 3),        # ragged row block (40 = 30 + 10), two pixel blocks
                 (3, 37, 64, 3, 64, 3, 3),        # three pixel blocks of 28, 28, 8
                 (2, 30, 40, 1, 64, 3, 3),        # C = 1 (85 pixels per accumulator)
                 (1, 33, 32, 1, 64, 5, 5),        # 5x5 taps: lane quarters overlap by 4 rows
                 (1, 19, 24, 4, 64, 3, 3),        # C = 4
                 (2, 20, 40, 3, 128, 3, 3),       # 128 filters: two 64-filter groups per dy row
                 (1, 12, 24, 1, 256, 3, 3),       # 256 filters: four groups, one dy row per weight-gradient tile
                 (1, 20, 40, 3, 64, 5, 5),        # 5x5x3: input gradient on the tensor cores, weight gradient has no tensor-core kernel (75 Hankel rows): refused
                 (1, 16, 24, 2, 64, 3, 3),        # C = 2
                 (1, 12, 24, 8, 64, 3, 3),        # C = 8: no tensor-core weight gradient (refused)
                 (1, 20, 40, 1, 64, 7, 7)]        # 7x7 taps: lane quarters overlap by 6 pixels, 6 replayed rows


@pytest.mark.parametrize("shape", BWD_TC_SHAPES)
def test_tensor_core_wgrad_and_dgrad_vs_oracle_and_fma_path(eng, pkg, shape):
    """The wgmma backward kernels (csrc/conv_wgrad_tc.cu, csrc/conv_dgrad_tc.cu; 64 filters) against the oracle on the same bf16-rounded operands, and
    against the FMA-pipe kernels of csrc/conv_bwd.cu (pcnn_conv_bwd_select).  fp32 accumulation everywhere:
    wgrad rel-L2 <= 1e-5 vs the oracle; dgrad |d| <= 2^-8 |ref| + 1e-3 (one bf16 rounding of the result)."""
    N, H, W, C, K, R, S = shape
    rng = np.random.default_rng(sum(shape) + 1)
    P, Q = H - R + 1, W - S + 1
    x = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(0, 1, (N, H, W, C)).astype(np.float32)))
    dy = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-1, 1, (N, P, Q, K)).astype(np.float32)))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    dw_ref = np.empty((K, R, S, C), np.float32)
    dx_ref = np.empty((N, H, W, C), np.float32)
    O.oracle().orc_conv_wgrad_nhwc(O.fp(x.reshape(-1)), O.fp(dy.reshape(-1)), O.fp(dw_ref.reshape(-1)), N, H, W, C, K, R, S)
    O.oracle().orc_conv_dgrad_nhwc(O.fp(dy.reshape(-1)), O.fp(f.reshape(-1)), O.fp(dx_ref.reshape(-1)), N, H, W, C, K, R, S)
    dxb, dyb, fd = eng.to_device(pkg.f32_to_bf16_bits(x)), eng.to_device(pkg.f32_to_bf16_bits(dy)), eng.to_device(f)
    res = {}
    import ctypes as C_
    info = (C_.c_int * 9)()
    assert pkg.lib().pcnn_conv_bwd_plan_info(N, H, W, C, K, R, S, info) == 0
    wgrad_tc, dgrad_tc = bool(info[0]), bool(info[4])
    assert dgrad_tc                                          # every shape of this list has a tensor-core input gradient
    try:
        for path in ("tc", "fma"):
            eng.conv_bwd_select(reference=(path == "fma"))
            launches0 = eng.launch_count()
            dw = eng.array((K, R, S, C))
            got_w = None
            if path == "fma" or wgrad_tc:
                eng.conv_wgrad(dxb, dyb, dw, N, H, W, C, K, R, S)
                got_w = dw.to_host()
                assert np.linalg.norm((got_w - dw_ref).astype(np.float64)) / np.linalg.norm(dw_ref.astype(np.float64)) <= 1e-5, path
                eng.conv_wgrad(dxb, dyb, dw, N, H, W, C, K, R, S)
                assert np.array_equal(dw.to_host().view(np.uint32), got_w.view(np.uint32)), path               # deterministic
            else:                                            # no tensor-core weight gradient for this shape: refused, not rerouted
                with pytest.raises(pkg.PcnnError, match="pcnn_conv_bwd_select"):
                    eng.conv_wgrad(dxb, dyb, dw, N, H, W, C, K, R, S)
            dxo = eng.array((N, H, W, C), np.uint16)
            eng.conv_dgrad(dyb, fd, dxo, N, H, W, C, K, R, S)
            got_x = pkg.bf16_bits_to_f32(dxo.to_host())
            assert np.all(np.abs(got_x - dx_ref) <= 2.0 ** -8 * np.abs(dx_ref) + 1e-3), path
            res[path] = (got_w, got_x, eng.launch_count() - launches0)
    finally:
        eng.conv_bwd_select(reference=False)
    # the two paths are different kernels (the dgrad launch counts differ: the tensor-core path also builds its filter variants)
    assert res["tc"][2] != res["fma"][2]
    if wgrad_tc:
        assert np.linalg.norm(res["tc"][0] - res["fma"][0]) / np.linalg.norm(res["fma"][0]) <= 1e-5


def test_tensor_core_dgrad_honours_row_and_image_pitch(eng, pkg):
    """dx written into a padded layout (row pitch 128 elements, 48 rows per image): pad elements keep their previous contents."""
    N, H, W, C, K, R, S = 2, 40, 40, 3, 64, 3, 3
    rng = np.random.default_rng(5)
    P, Q = H - R + 1, W - S + 1
    dy = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-1, 1, (N, P, Q, K)).astype(np.float32)))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    dx_ref = np.empty((N, H, W, C), np.float32)
    O.oracle().orc_conv_dgrad_nhwc(O.fp(dy.reshape(-1)), O.fp(f.reshape(-1)), O.fp(dx_ref.reshape(-1)), N, H, W, C, K, R, S)
    pitch, rows = 128, 48
    canvas = np.full((N, rows, pitch), 0x4242, np.uint16)
    dxo = eng.to_device(canvas)
    eng.conv_dgrad(eng.to_device(pkg.f32_to_bf16_bits(dy)), eng.to_device(f), dxo, N, H, W, C, K, R, S, row_pitch=pitch, image_rows=rows)
    out = dxo.to_host().reshape(N, rows, pitch)
    got = pkg.bf16_bits_to_f32(out[:, :H, :W * C].reshape(N, H, W, C))
    assert np.all(np.abs(got - dx_ref) <= 2.0 ** -8 * np.abs(dx_ref) + 1e-3)
    assert np.all(out[:, H:, :] == 0x4242) and np.all(out[:, :, W * C:] == 0x4242)


def test_measurement_probes_report_sane_rates(eng, pkg):
    """pcnn_measure_mma_rate / pcnn_measure_tma_read (the tables DESIGN.md 3.7 designs against): one small M = 128 wgmma product costs
    tens of clocks, not hundreds; a TMA pipeline streams well above 1 TB/s with contiguous boxes and with the row-gather boxes alike
    (on H100 both reach the same HBM ceiling: 2,812 vs 2,814 GB/s measured, so neither is required to beat the other)."""
    clk = eng.measure_mma_rate(128, 64, 0, 0, 1, 2000)
    assert 30.0 < clk < 200.0, clk
    assert eng.measure_mma_rate(128, 256, 0, 0, 1, 2000) > 1.5 * clk         # N = 256 is bound by the tensor pipe, not by issue
    N, P, Q = 16, 222, 222
    buf = eng.array((N, P, Q, 64), np.uint16)
    contiguous = eng.measure_tma_read(buf, N, P, Q, 3, 5)
    gather = eng.measure_tma_read(buf, N, P, Q, 2, 5)
    assert contiguous > 1000.0 and gather > 1000.0, (contiguous, gather)


def test_same_padding_convolution_through_pad_and_crop(eng, pkg):
    """SURVEY.md 8f row 4: a 'same' (zero padded) 3x3 convolution, its weight gradient and its input gradient through
    pcnn_pad_nhwc_bf16 / pcnn_crop_nhwc_bf16 around the valid-padding tensor-core kernels, against the oracle evaluated on
    the host-padded tensors (tolerances as in the valid-padding tests)."""
    N, H, W, C, K, R, S, pad = 2, 30, 40, 3, 64, 3, 3, 1
    Hp, Wp = H + 2 * pad, W + 2 * pad
    rng = np.random.default_rng(11)
    x = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(0, 1, (N, H, W, C)).astype(np.float32)))
    f = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-0.5, 0.5, (K, R, S, C)).astype(np.float32)))
    dy = pkg.bf16_bits_to_f32(pkg.f32_to_bf16_bits(rng.uniform(-1, 1, (N, H, W, K)).astype(np.float32)))      # same padding: P x Q = H x W
    xp = np.zeros((N, Hp, Wp, C), np.float32)
    xp[:, pad:pad + H, pad:pad + W, :] = x
    y_ref = np.empty((N, H, W, K), np.float32)
    dw_ref = np.empty((K, R, S, C), np.float32)
    dxp_ref = np.empty((N, Hp, Wp, C), np.float32)
    zero_b = np.zeros(K, np.float32)
    O.oracle().orc_conv_fwd_nhwc(O.fp(xp.reshape(-1)), O.fp(f.reshape(-1)), O.fp(zero_b), O.fp(y_ref.reshape(-1)), N, Hp, Wp, C, K, R, S)
    O.oracle().orc_conv_wgrad_nhwc(O.fp(xp.reshape(-1)), O.fp(dy.reshape(-1)), O.fp(dw_ref.reshape(-1)), N, Hp, Wp, C, K, R, S)
    O.oracle().orc_conv_dgrad_nhwc(O.fp(dy.reshape(-1)), O.fp(f.reshape(-1)), O.fp(dxp_ref.reshape(-1)), N, Hp, Wp, C, K, R, S)
    # device: pad (row pitch rounded to 8 elements for the forward plan), forward, backward, crop
    pitch = (Wp * C + 7) // 8 * 8
    dxs = eng.to_device(pkg.f32_to_bf16_bits(x))
    canvas = eng.to_device(np.full((N, Hp, pitch), 0x4242, np.uint16))                       # pad kernel must overwrite the garbage
    eng.pad_nhwc(dxs, canvas, N, H, W, C, pad, pad, dst_row_pitch=pitch)
    got_canvas = canvas.to_host().reshape(N, Hp, pitch)
    assert np.array_equal(got_canvas[:, :, :Wp * C].reshape(N, Hp, Wp, C), pkg.f32_to_bf16_bits(xp))
    assert np.all(got_canvas[:, :, Wp * C:] == 0)
    plan = pkg.ConvPlan(eng, N, Hp, Wp, C, K, R, S, f, None, act=0, row_pitch=pitch)
    yd = eng.array((N, H, W, K), np.uint16)
    plan.fwd(canvas, yd)
    got_y = pkg.bf16_bits_to_f32(yd.to_host())
    plan.close()
    assert np.all(np.abs(got_y - y_ref) <= 2.0 ** -8 * np.abs(y_ref) + 1e-3)
    dyd = eng.to_device(pkg.f32_to_bf16_bits(dy))
    dw = eng.array((K, R, S, C))
    eng.conv_wgrad(canvas, dyd, dw, N, Hp, Wp, C, K, R, S, row_pitch=pitch)
    assert np.linalg.norm((dw.to_host() - dw_ref).astype(np.float64)) / np.linalg.norm(dw_ref.astype(np.float64)) <= 1e-5
    dxp = eng.array((N, Hp, Wp, C), np.uint16)
    eng.conv_dgrad(dyd, eng.to_device(f), dxp, N, Hp, Wp, C, K, R, S)
    dxc = eng.array((N, H, W, C), np.uint16)
    eng.crop_nhwc(dxp, dxc, N, H, W, C, pad, pad)
    got_dx = pkg.bf16_bits_to_f32(dxc.to_host())
    ref_dx = dxp_ref[:, pad:pad + H, pad:pad + W, :]
    assert np.all(np.abs(got_dx - ref_dx) <= 2.0 ** -8 * np.abs(ref_dx) + 1e-3)
