"""Engine: a thin object wrapper over one pcnn_ctx.  Method names follow include/pcnn.h minus the pcnn_ prefix, which
in turn follow /root/reference/Sequential/layer.h and Main.cpp (fp_c1, bp_weight_c1, learn, test ...)."""
import ctypes as C
import math
from typing import NamedTuple, Optional

import numpy as np

from ._lib import (F32, NPARAM, OPTIM_ADAMW, OPTIM_SGD, TEST_SET, TRAIN_SET, U8, OptimConfig, OptimTensor, PcnnError, augment_info,
                   augment_resized_info, RESIZE_TRAIN, RESIZE_EVAL, augment_trivial_info, TRIVIAL_NONE, TRIVIAL_NEAREST, TRIVIAL_BILINEAR,
                   attention_info, avgpool_nhwc_info, batchnorm_nhwc_info, channel_stats, check, conv_layer_family, conv_transpose_info, upsample_bilinear_info, dropout_info, dwconv_info, gconv_info, global_avgpool_nhwc_info, groupnorm_nhwc_info, lib,
                   linear_info, maxpool_nhwc_info, pixel_shuffle_info, LOSS_MSE, gaussian_latent_info,
                   se_scale_nhwc_info, ACT_RELU, ACT_SIGMOID, ACT_SILU, ACT_HARDSWISH, ACT_RELU6)

PREACT_CODES = (ACT_SILU, ACT_HARDSWISH, ACT_RELU6)   # the normalizations' codes whose backward recomputes the pre-activation
MIX_MIXUP, MIX_CUTMIX = 1, 2                         # pcnn_augment_mix_u8_bf16's modes


def _pixel_type(arr_or_dtype):
    dt = np.dtype(getattr(arr_or_dtype, "dtype", arr_or_dtype))
    if dt == np.uint8:
        return U8
    if dt == np.float32:
        return F32
    raise PcnnError("pixel_type", -1, f"images must be uint8 or float32, got {dt}")


class DeviceArray:
    """A device buffer obtained from pcnn_malloc (zero-initialised like the reference's `new float[n]()`)."""

    def __init__(self, engine, shape, dtype=np.float32):
        self.engine = engine
        self.shape = tuple(int(s) for s in (shape if isinstance(shape, (tuple, list)) else (shape,)))
        self.dtype = np.dtype(dtype)
        self.nbytes = int(np.prod(self.shape, dtype=np.int64)) * self.dtype.itemsize
        p = C.c_void_p()
        check("pcnn_malloc", lib().pcnn_malloc(engine.ctx, C.byref(p), self.nbytes))
        self.ptr = p.value

    @classmethod
    def from_host(cls, engine, host):
        host = np.ascontiguousarray(host)
        d = cls(engine, host.shape, host.dtype)
        d.copy_from(host)
        return d

    def copy_from(self, host):
        host = np.ascontiguousarray(host, self.dtype)
        assert host.nbytes == self.nbytes, (host.shape, self.shape)
        check("pcnn_h2d", lib().pcnn_h2d(self.engine.ctx, self.ptr, host.ctypes.data, self.nbytes))
        return self

    def to_host(self):
        out = np.empty(self.shape, self.dtype)
        check("pcnn_d2h", lib().pcnn_d2h(self.engine.ctx, out.ctypes.data, self.ptr, self.nbytes))
        return out

    def zero(self):
        check("pcnn_memset0", lib().pcnn_memset0(self.engine.ctx, self.ptr, self.nbytes))

    def free(self):
        if self.ptr and self.engine.ctx:
            lib().pcnn_free(self.engine.ctx, self.ptr)
        self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _p(x):
    """device pointer of a DeviceArray / raw int / torch tensor (data_ptr) / None"""
    if x is None:
        return None
    if isinstance(x, DeviceArray):
        return x.ptr
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    return int(x)


class Engine:
    def __init__(self, device=-1, stream=None):
        self.ctx = None
        ctx = C.c_void_p()
        check("pcnn_create", lib().pcnn_create(C.byref(ctx), int(device), stream))
        self.ctx = ctx

    def close(self):
        if self.ctx:
            lib().pcnn_destroy(self.ctx)
            self.ctx = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _call(self, name, *args):
        check(name, getattr(lib(), name)(self.ctx, *args))

    # ------------------------------------------------------------------ context / parameters
    def sync(self):
        self._call("pcnn_sync")

    def device_info(self):
        sm, ma, mi, hb = C.c_int(), C.c_int(), C.c_int(), C.c_size_t()
        self._call("pcnn_device_info", C.byref(sm), C.byref(ma), C.byref(mi), C.byref(hb))
        return dict(sm_count=sm.value, cc=(ma.value, mi.value), hbm_bytes=hb.value)

    def array(self, shape, dtype=np.float32):
        return DeviceArray(self, shape, dtype)

    def to_device(self, host):
        return DeviceArray.from_host(self, host)

    def set_params(self, p):
        p = np.ascontiguousarray(p, np.float32)
        assert p.size == NPARAM
        self._call("pcnn_set_params", p.ctypes.data)

    def get_params(self):
        p = np.empty(NPARAM, np.float32)
        self._call("pcnn_get_params", p.ctypes.data)
        return p

    def get_grads(self):
        g = np.empty(NPARAM, np.float32)
        self._call("pcnn_get_grads", g.ctypes.data)
        return g

    def params_dev(self):
        p = C.c_void_p()
        self._call("pcnn_params_dev", C.byref(p))
        return p.value

    def set_learning_rate(self, dt):
        self._call("pcnn_set_learning_rate", float(dt))

    def save_params(self, path):
        self._call("pcnn_save_params", str(path).encode())

    def load_params(self, path):
        self._call("pcnn_load_params", str(path).encode())

    def err_sum(self, reset=False):
        s = C.c_double()
        self._call("pcnn_err_sum", C.byref(s), 1 if reset else 0)
        return s.value

    def launch_count(self):
        n = C.c_long()
        self._call("pcnn_launch_count", C.byref(n))
        return n.value

    # ------------------------------------------------------------------ per-operator API (layer.h names)
    def apply_step_function(self, inp, out, n):
        self._call("pcnn_apply_step_function", _p(inp), _p(out), int(n))

    def makeError(self, err, out, Y, n=10):
        self._call("pcnn_make_error", _p(err), _p(out), int(Y), int(n))

    def makeError_batch(self, err, out, labels, B):
        self._call("pcnn_make_error_batch", _p(err), _p(out), _p(labels), int(B))

    def apply_grad(self, w, g, n):
        self._call("pcnn_apply_grad", _p(w), _p(g), int(n))

    def apply_grad_scaled(self, w, g, n, step):
        """w += step * g over n fp32 elements (__fmul_rn, then __fadd_rn)"""
        self._call("pcnn_apply_grad_scaled", _p(w), _p(g), int(n), float(step))

    def vectorNorm(self, v, n, B, norms):
        self._call("pcnn_vector_norm", _p(v), int(n), int(B), _p(norms))

    def fp_c1(self, inp, pre, w, b, B=1):
        self._call("pcnn_fp_c1", _p(inp), _p(pre), _p(w), _p(b), int(B))

    def fp_s1(self, inp, pre, w, b, B=1):
        self._call("pcnn_fp_s1", _p(inp), _p(pre), _p(w), _p(b), int(B))

    def fp_preact_f(self, inp, pre, w, B=1):
        self._call("pcnn_fp_preact_f", _p(inp), _p(pre), _p(w), int(B))

    def fp_bias_f(self, pre, b, B=1):
        self._call("pcnn_fp_bias_f", _p(pre), _p(b), int(B))

    def bp_weight_f(self, dw, dpre, pout, B=1):
        self._call("pcnn_bp_weight_f", _p(dw), _p(dpre), _p(pout), int(B))

    def bp_bias_f(self, bias, dpre, B=1):
        self._call("pcnn_bp_bias_f", _p(bias), _p(dpre), int(B))

    def bp_output_s1(self, dout, nw, ndpre, B=1):
        self._call("pcnn_bp_output_s1", _p(dout), _p(nw), _p(ndpre), int(B))

    def bp_preact_s1(self, dpre, dout, pre, B=1):
        self._call("pcnn_bp_preact_s1", _p(dpre), _p(dout), _p(pre), int(B))

    def bp_weight_s1(self, dw, dpre, pout, B=1):
        self._call("pcnn_bp_weight_s1", _p(dw), _p(dpre), _p(pout), int(B))

    def bp_bias_s1(self, bias, dpre, B=1):
        self._call("pcnn_bp_bias_s1", _p(bias), _p(dpre), int(B))

    def bp_output_c1(self, dout, nw, ndpre, B=1):
        self._call("pcnn_bp_output_c1", _p(dout), _p(nw), _p(ndpre), int(B))

    def bp_preact_c1(self, dpre, dout, pre, B=1):
        self._call("pcnn_bp_preact_c1", _p(dpre), _p(dout), _p(pre), int(B))

    def bp_weight_c1(self, dw, dpre, pout, B=1):
        self._call("pcnn_bp_weight_c1", _p(dw), _p(dpre), _p(pout), int(B))

    def bp_bias_c1(self, bias, dpre, B=1):
        self._call("pcnn_bp_bias_c1", _p(bias), _p(dpre), int(B))

    # ------------------------------------------------------------------ data + fused path (Main.cpp names)
    def dataset_upload(self, split, images, labels):
        images = np.ascontiguousarray(images)
        labels = np.ascontiguousarray(labels, np.uint8)
        n = labels.shape[0]
        assert images.size == n * 784
        self._call("pcnn_dataset_upload", int(split), images.ctypes.data, _pixel_type(images), labels.ctypes.data, n)

    def dataset_bind(self, split, images_dev, pixel_type, labels_dev, n):
        self._call("pcnn_dataset_bind", int(split), _p(images_dev), int(pixel_type), _p(labels_dev), int(n))

    def train_step(self, first, B):
        self._call("pcnn_train_step", int(first), int(B))

    def train_steps(self, first, B, nsteps):
        self._call("pcnn_train_steps", int(first), int(B), int(nsteps))

    def train_steps_prepare(self, B, nsteps):
        self._call("pcnn_train_steps_prepare", int(B), int(nsteps))

    def train_step_dev(self, images_dev, pixel_type, labels_dev, B):
        self._call("pcnn_train_step_dev", _p(images_dev), int(pixel_type), _p(labels_dev), int(B))

    def train_step_host(self, images, labels):
        images = np.ascontiguousarray(images)
        labels = np.ascontiguousarray(labels, np.uint8)
        e = C.c_float()
        self._call("pcnn_train_step_host", images.ctypes.data, _pixel_type(images), labels.ctypes.data,
                   labels.shape[0], C.byref(e))
        return e.value

    def compute_grads(self, images_dev, pixel_type, labels_dev, B):
        self._call("pcnn_compute_grads", _p(images_dev), int(pixel_type), _p(labels_dev), int(B))

    def learn(self, B=1, epochs=1):
        e = C.c_float()
        self._call("pcnn_learn", int(B), int(epochs), C.byref(e))
        return e.value

    def learn_host(self, images, labels, B=1, epochs=1):
        images = np.ascontiguousarray(images)
        labels = np.ascontiguousarray(labels, np.uint8)
        e = C.c_float()
        self._call("pcnn_learn_host", images.ctypes.data, _pixel_type(images), labels.ctypes.data, labels.shape[0],
                   int(B), int(epochs), C.byref(e))
        return e.value

    def forward_batch(self, images_dev, pixel_type, B, f_out_dev=None, pred_dev=None):
        self._call("pcnn_forward_batch", _p(images_dev), int(pixel_type), int(B), _p(f_out_dev), _p(pred_dev))

    def test(self):
        w = C.c_long()
        self._call("pcnn_test", C.byref(w))
        return w.value

    def step_errs(self):
        n = C.c_long()
        self._call("pcnn_step_errs", None, 0, C.byref(n))
        out = np.empty(n.value, np.float32)
        self._call("pcnn_step_errs", out.ctypes.data, n.value, C.byref(n))
        return out

    def time_fused_kernel(self, B, iters):
        ms = C.c_float()
        self._call("pcnn_time_fused_kernel", int(B), int(iters), C.byref(ms))
        return ms.value

    def measure_fp32_peak(self):
        t = C.c_float()
        self._call("pcnn_measure_fp32_peak", C.byref(t))
        return t.value

    def measure_mma_rate(self, M, N, a_mn=0, b_mn=0, nacc=1, reps=2000):
        t = C.c_float()
        self._call("pcnn_measure_mma_rate", int(M), int(N), int(a_mn), int(b_mn), int(nacc), int(reps), C.byref(t))
        return t.value

    def measure_tma_read(self, dev_bf16, N, P, Q, mode, iters=10):
        t = C.c_float()
        self._call("pcnn_measure_tma_read", _p(dev_bf16), int(N), int(P), int(Q), int(mode), int(iters), C.byref(t))
        return t.value

    def measure_tma_write(self, dev_bf16, N, P, H, row_elems, mode, hot=0, iters=10):
        t = C.c_float()
        self._call("pcnn_measure_tma_write", _p(dev_bf16), int(N), int(P), int(H), int(row_elems), int(mode), int(hot), int(iters), C.byref(t))
        return t.value

    # ------------------------------------------------------------------ data parallel
    @staticmethod
    def comm_unique_id():
        buf = (C.c_char * 256)()
        n = C.c_size_t()
        check("pcnn_comm_unique_id", lib().pcnn_comm_unique_id(buf, C.byref(n)))
        return bytes(buf[: n.value])

    def comm_init_rank(self, uid, rank, world):
        self._call("pcnn_comm_init_rank", C.c_char_p(uid), int(rank), int(world))

    def comm_destroy(self):
        self._call("pcnn_comm_destroy")

    def allreduce_grads(self):
        self._call("pcnn_allreduce_grads")

    def p2p_export(self):
        buf = (C.c_char * 128)()
        n = C.c_size_t()
        self._call("pcnn_p2p_export", buf, C.byref(n))
        return bytes(buf[: n.value])

    def p2p_attach(self, handles, rank, world):
        """handles: list of the `world` byte strings returned by every rank's p2p_export(), in rank order"""
        blob = b"".join(handles)
        self._call("pcnn_p2p_attach", C.c_char_p(blob), int(rank), int(world))

    def p2p_detach(self):
        self._call("pcnn_p2p_detach")

    def set_step_mode(self, mode):
        self._call("pcnn_set_step_mode", int(mode))

    def persist_trace_ctas(self, ctas):
        out = np.zeros((int(ctas), 8), np.int64)
        self._call("pcnn_persist_trace_ctas", out.ctypes.data, int(ctas))
        return out

    def persist_info(self):
        out = np.zeros(6, np.int32)
        self._call("pcnn_persist_info", out.ctypes.data)
        return {"grid": int(out[0]), "cluster": int(out[1]), "cta_capacity": int(out[2]), "cta_capacity_clustered": int(out[3]),
                "cluster_size_used_when_possible": int(out[4]), "cooperative": bool(out[5] & 1), "direct_exchange": bool(out[5] & 2),
                "images_per_cta": 2 if out[5] & 4 else 1}

    def persist_tune(self, max_cluster=0):
        self._call("pcnn_persist_tune", int(max_cluster))

    def persist_trace_arm(self):
        self._call("pcnn_persist_trace", None, 0)

    def persist_trace_read(self, steps=256):
        out = np.zeros((steps, 6), np.int64)
        self._call("pcnn_persist_trace", out.ctypes.data, int(steps))
        return out

    # ------------------------------------------------------------------ extension ops
    def maxpool_fwd(self, inp, out, argmax, planes, H, W, k):
        self._call("pcnn_maxpool_fwd", _p(inp), _p(out), _p(argmax), int(planes), int(H), int(W), int(k))

    def maxpool_bwd(self, dout, argmax, din, planes, H, W, k):
        self._call("pcnn_maxpool_bwd", _p(dout), _p(argmax), _p(din), int(planes), int(H), int(W), int(k))

    # LeNet-5-style variant (second convolution layer); all arguments are DeviceArrays
    def l5_compute_grads(self, params, images, pixel_type, labels, B, grads):
        self._call("pcnn_l5_compute_grads", _p(params), _p(images), int(pixel_type), _p(labels), int(B), _p(grads))

    def l5_train_step(self, params, images, pixel_type, labels, B, grads=None):
        self._call("pcnn_l5_train_step", _p(params), _p(images), int(pixel_type), _p(labels), int(B), _p(grads) if grads is not None else None)

    def l5_forward(self, params, images, pixel_type, B, f_out):
        self._call("pcnn_l5_forward", _p(params), _p(images), int(pixel_type), int(B), _p(f_out))

    def conv_bwd_select(self, reference=False):
        """reference=True: the FMA-pipe reference kernels for every shape (explicit opt-in); False: tensor cores only"""
        self._call("pcnn_conv_bwd_select", 1 if reference else 0)

    def conv_wgrad(self, x_bf16, dy_bf16, dw_f32, N, H, W, Cin, K, R, S, row_pitch=0, image_rows=0, stride=1):
        self._call("pcnn_conv_wgrad_strided", _p(x_bf16), _p(dy_bf16), _p(dw_f32), N, H, W, Cin, K, R, S, int(stride), int(row_pitch),
                   int(image_rows))

    def conv_dgrad(self, dy_bf16, filt_f32, dx_bf16, N, H, W, Cin, K, R, S, row_pitch=0, image_rows=0, stride=1):
        self._call("pcnn_conv_dgrad_strided", _p(dy_bf16), _p(filt_f32), _p(dx_bf16), N, H, W, Cin, K, R, S, int(stride), int(row_pitch),
                   int(image_rows))

    def conv_wide_wgrad(self, x_bf16, dy_bf16, dw_f32, N, H, W, Cin, K, R, S, row_pitch=None, image_rows=0, stride=1, padding=(0, 0),
                        dilation=(1, 1)):
        """weight gradient of WideConvPlan's forward (pcnn_conv_wide_wgrad, or pcnn_conv_wide_wgrad_padded for a zero padding
        (pad_h, pad_w) other than (0, 0), or pcnn_conv_wide_wgrad_dilated for a dilation other than (1, 1)); row_pitch None =
        W*Cin rounded up to 8, as the plan"""
        pitch = (W * Cin + 7) // 8 * 8 if row_pitch is None else row_pitch
        ph, pw = (int(v) for v in padding)
        dh, dw = (int(v) for v in dilation)
        if (dh, dw) != (1, 1):
            self._call("pcnn_conv_wide_wgrad_dilated", _p(x_bf16), _p(dy_bf16), _p(dw_f32), N, H, W, Cin, K, R, S, int(stride), ph, pw,
                       dh, dw, int(pitch), int(image_rows))
        elif (ph, pw) == (0, 0):
            self._call("pcnn_conv_wide_wgrad", _p(x_bf16), _p(dy_bf16), _p(dw_f32), N, H, W, Cin, K, R, S, int(stride), int(pitch),
                       int(image_rows))
        else:
            self._call("pcnn_conv_wide_wgrad_padded", _p(x_bf16), _p(dy_bf16), _p(dw_f32), N, H, W, Cin, K, R, S, int(stride), ph, pw,
                       int(pitch), int(image_rows))

    def conv_wide_dgrad(self, dy_bf16, filt_f32, dx_bf16, N, H, W, Cin, K, R, S, row_pitch=None, image_rows=0, stride=1, padding=(0, 0),
                        dilation=(1, 1)):
        """input gradient of WideConvPlan's forward (pcnn_conv_wide_dgrad, or pcnn_conv_wide_dgrad_padded for a zero padding
        (pad_h, pad_w) other than (0, 0), or pcnn_conv_wide_dgrad_dilated for a dilation other than (1, 1)) into dx in x's layout"""
        pitch = (W * Cin + 7) // 8 * 8 if row_pitch is None else row_pitch
        ph, pw = (int(v) for v in padding)
        dh, dw = (int(v) for v in dilation)
        if (dh, dw) != (1, 1):
            self._call("pcnn_conv_wide_dgrad_dilated", _p(dy_bf16), _p(filt_f32), _p(dx_bf16), N, H, W, Cin, K, R, S, int(stride), ph, pw,
                       dh, dw, int(pitch), int(image_rows))
        elif (ph, pw) == (0, 0):
            self._call("pcnn_conv_wide_dgrad", _p(dy_bf16), _p(filt_f32), _p(dx_bf16), N, H, W, Cin, K, R, S, int(stride), int(pitch),
                       int(image_rows))
        else:
            self._call("pcnn_conv_wide_dgrad_padded", _p(dy_bf16), _p(filt_f32), _p(dx_bf16), N, H, W, Cin, K, R, S, int(stride), ph, pw,
                       int(pitch), int(image_rows))

    def conv_bias_act_bwd(self, y, dy, dpre, db, pixels, K, act):
        """pcnn_conv_bias_act_bwd: dpre = bf16(dy * y * (1 - y)) at act 1 (ACT_SIGMOID), dpre = (y <= 0 ? +0 : dy) at act 3
        (ACT_RELU; dy's bits pass through, a NaN y passes dy); dpre may be dy itself.  db[k] = sum of dpre (of dy at act 0) over the
        pixels; dpre None at act 0, db None for a layer without bias"""
        self._call("pcnn_conv_bias_act_bwd", _p(y), _p(dy), _p(dpre), _p(db), int(pixels), int(K), int(act))

    def maxpool_nhwc_fwd(self, x, y, argmax, N, H, W, Cin, R, S, stride, padding=(0, 0), row_pitch=None, image_rows=0):
        """pcnn_maxpool_nhwc_bf16_fwd: x dense bf16 [N][H][W][C] -> y [N][image_rows][row_pitch] (P x Q pixels of C channels per
        image) and the uint8 argmax r*S + s [N][P][Q][C] (None for inference); row_pitch None = Q*C rounded up to 8, image_rows 0 = P"""
        ph, pw = (int(v) for v in padding)
        self._call("pcnn_maxpool_nhwc_bf16_fwd", _p(x), _p(y), _p(argmax), int(N), int(H), int(W), int(Cin), int(R), int(S), int(stride),
                   ph, pw, int(row_pitch or 0), int(image_rows))

    def maxpool_nhwc_bwd(self, dy, argmax, dx, N, H, W, Cin, R, S, stride, padding=(0, 0), row_pitch=None, image_rows=0):
        """pcnn_maxpool_nhwc_bf16_bwd: dy in y's layout and the forward's argmax -> dx dense bf16 [N][H][W][C], every element written"""
        ph, pw = (int(v) for v in padding)
        self._call("pcnn_maxpool_nhwc_bf16_bwd", _p(dy), _p(argmax), _p(dx), int(N), int(H), int(W), int(Cin), int(R), int(S), int(stride),
                   ph, pw, int(row_pitch or 0), int(image_rows))

    def avgpool_nhwc_fwd(self, x, y, N, H, W, Cin, R, S, stride, padding=(0, 0), count_include_pad=True, row_pitch=None, image_rows=0):
        """pcnn_avgpool_nhwc_bf16_fwd: x dense bf16 [N][H][W][C] -> y [N][image_rows][row_pitch], each window's in-image sum over
        R*S (count_include_pad) or over its in-image positions; row_pitch None = Q*C rounded up to 8, image_rows 0 = P"""
        ph, pw = (int(v) for v in padding)
        self._call("pcnn_avgpool_nhwc_bf16_fwd", _p(x), _p(y), int(N), int(H), int(W), int(Cin), int(R), int(S), int(stride), ph, pw,
                   int(count_include_pad), int(row_pitch or 0), int(image_rows))

    def avgpool_nhwc_bwd(self, dy, dx, N, H, W, Cin, R, S, stride, padding=(0, 0), count_include_pad=True, row_pitch=None, image_rows=0):
        """pcnn_avgpool_nhwc_bf16_bwd: dy in y's layout -> dx dense bf16 [N][H][W][C], every element written"""
        ph, pw = (int(v) for v in padding)
        self._call("pcnn_avgpool_nhwc_bf16_bwd", _p(dy), _p(dx), int(N), int(H), int(W), int(Cin), int(R), int(S), int(stride), ph, pw,
                   int(count_include_pad), int(row_pitch or 0), int(image_rows))

    def global_avgpool_nhwc_fwd(self, x, y, N, H, W, Cin, row_pitch=None):
        """pcnn_global_avgpool_nhwc_bf16_fwd: x dense bf16 [N][H][W][C] -> y [N][row_pitch], the mean over the H*W pixels;
        row_pitch None = C rounded up to 8"""
        self._call("pcnn_global_avgpool_nhwc_bf16_fwd", _p(x), _p(y), int(N), int(H), int(W), int(Cin), int(row_pitch or 0))

    def global_avgpool_nhwc_bwd(self, dy, dx, N, H, W, Cin, row_pitch=None):
        """pcnn_global_avgpool_nhwc_bf16_bwd: dy [N][row_pitch] -> dx dense bf16 [N][H][W][C] = dy / (H*W) at every pixel"""
        self._call("pcnn_global_avgpool_nhwc_bf16_bwd", _p(dy), _p(dx), int(N), int(H), int(W), int(Cin), int(row_pitch or 0))

    def batchnorm_fwd(self, x, y, pixels, C, gamma, beta, running_mean=None, running_var=None, save_mean=None, save_rstd=None, r=None,
                      act=0, training=True, eps=1e-5, momentum=0.1):
        """pcnn_batchnorm_nhwc_bf16_fwd: y = bf16(act((x - mean) * rstd * gamma + beta (+ r))) over dense bf16 [pixels][C].
        training: batch statistics into save_mean / save_rstd and, when given, the running statistics updated with momentum;
        eval: the running statistics.  act ACT_NONE, ACT_RELU, ACT_SILU, ACT_HARDSWISH or ACT_RELU6"""
        self._call("pcnn_batchnorm_nhwc_bf16_fwd", _p(x), _p(r), _p(y), int(pixels), int(C), int(act), 1 if training else 0, float(eps),
                   float(momentum), _p(gamma), _p(beta), _p(running_mean), _p(running_var), _p(save_mean), _p(save_rstd))

    def batchnorm_bwd(self, x, y, dy, gamma, save_mean, save_rstd, dx, dgamma, dbeta, pixels, C, act=0, dy2=None, dr=None):
        """pcnn_batchnorm_nhwc_bf16_bwd of a training forward: g = bf16(act'(dy (+ dy2))), dbeta = sum g, dgamma = sum g * xhat,
        dx (may be dy itself) and, when given, dr = g (the gradient of the forward's residual input)"""
        self._call("pcnn_batchnorm_nhwc_bf16_bwd", _p(x), _p(y), _p(dy), _p(dy2), _p(gamma), _p(save_mean), _p(save_rstd), _p(dx), _p(dr),
                   _p(dgamma), _p(dbeta), int(pixels), int(C), int(act))

    def batchnorm_bwd_preact(self, x, dy, gamma, beta, save_mean, save_rstd, dx, dgamma, dbeta, pixels, C, act, r=None, dy2=None,
                             dr=None):
        """pcnn_batchnorm_nhwc_bf16_bwd_preact of a training forward at ACT_SILU, ACT_HARDSWISH or ACT_RELU6: as batchnorm_bwd, with
        g = bf16(act'(v) * (dy (+ dy2))) taken at the pre-activation v recomputed from x, the saved statistics, gamma, beta and r (the
        forward's r, unchanged, or None if it had none) instead of from y"""
        self._call("pcnn_batchnorm_nhwc_bf16_bwd_preact", _p(x), _p(r), _p(dy), _p(dy2), _p(gamma), _p(beta), _p(save_mean), _p(save_rstd),
                   _p(dx), _p(dr), _p(dgamma), _p(dbeta), int(pixels), int(C), int(act))

    def groupnorm_fwd(self, x, y, N, HW, C, G, gamma, beta, save_mean, save_rstd, r=None, act=0, eps=1e-5):
        """pcnn_groupnorm_nhwc_bf16_fwd: y = bf16(act((x - mean) * rstd * gamma + beta (+ r))) over dense bf16 [N][HW][C], mean and
        rstd those of each (image, group of C / G channels), written to save_mean / save_rstd [N][G].  act ACT_NONE, ACT_RELU,
        ACT_SILU, ACT_HARDSWISH or ACT_RELU6"""
        self._call("pcnn_groupnorm_nhwc_bf16_fwd", _p(x), _p(r), _p(y), int(N), int(HW), int(C), int(G), int(act), float(eps), _p(gamma),
                   _p(beta), _p(save_mean), _p(save_rstd))

    def groupnorm_bwd(self, x, y, dy, gamma, save_mean, save_rstd, dx, dgamma, dbeta, dstat, N, HW, C, G, act=0, dy2=None, dr=None):
        """pcnn_groupnorm_nhwc_bf16_bwd at ACT_NONE or ACT_RELU: g = bf16(act'(dy (+ dy2))), dbeta = sum g, dgamma = sum g * xhat over
        the batch, dstat [2][N][G] = the group sums A = sum gamma * g and B = sum gamma * g * xhat, dx (may be dy itself) and, when
        given, dr = g"""
        self._call("pcnn_groupnorm_nhwc_bf16_bwd", _p(x), _p(y), _p(dy), _p(dy2), _p(gamma), _p(save_mean), _p(save_rstd), _p(dx), _p(dr),
                   _p(dgamma), _p(dbeta), _p(dstat), int(N), int(HW), int(C), int(G), int(act))

    def groupnorm_bwd_preact(self, x, dy, gamma, beta, save_mean, save_rstd, dx, dgamma, dbeta, dstat, N, HW, C, G, act, r=None, dy2=None,
                             dr=None):
        """pcnn_groupnorm_nhwc_bf16_bwd_preact at ACT_SILU, ACT_HARDSWISH or ACT_RELU6: as groupnorm_bwd, with g taken at the
        pre-activation recomputed from x, the saved statistics, gamma, beta and r (the forward's r, unchanged, or None)"""
        self._call("pcnn_groupnorm_nhwc_bf16_bwd_preact", _p(x), _p(r), _p(dy), _p(dy2), _p(gamma), _p(beta), _p(save_mean), _p(save_rstd),
                   _p(dx), _p(dr), _p(dgamma), _p(dbeta), _p(dstat), int(N), int(HW), int(C), int(G), int(act))

    def attention_fwd(self, q, k, v, o, lse, N, T, heads, d, ld=None, scale=None):
        """pcnn_attention_bf16_fwd: o = softmax(scale q k^T) v per image and head over T tokens, lse [N][heads][T] its logsumexp.  q,
        k and v are bf16 rows of ld elements (default heads * d), head j at columns j d; o is dense [N][T][heads][d].  scale None =
        1 / sqrt(d)"""
        self._call("pcnn_attention_bf16_fwd", _p(q), _p(k), _p(v), int(N), int(T), int(heads), int(d), int(heads * d if ld is None else ld),
                   float(1.0 / math.sqrt(d) if scale is None else scale), _p(o), _p(lse))

    def attention_bwd(self, q, k, v, o, dout, lse, dq, dk, dv, N, T, heads, d, ld=None, ld_g=None, scale=None):
        """pcnn_attention_bf16_bwd: dq, dk and dv (rows of ld_g elements, default ld) of the forward that wrote o and lse, given
        dout [N][T][heads][d]; they may be the column blocks of one fused buffer"""
        ld = int(heads * d if ld is None else ld)
        self._call("pcnn_attention_bf16_bwd", _p(q), _p(k), _p(v), _p(o), _p(dout), _p(lse), int(N), int(T), int(heads), int(d), ld,
                   float(1.0 / math.sqrt(d) if scale is None else scale), _p(dq), _p(dk), _p(dv), int(ld if ld_g is None else ld_g))

    def pad_nhwc(self, src_bf16, dst_bf16, N, H, W, Cin, pad_h, pad_w, dst_row_pitch=0, dst_image_rows=0):
        self._call("pcnn_pad_nhwc_bf16", _p(src_bf16), _p(dst_bf16), N, H, W, Cin, int(pad_h), int(pad_w), int(dst_row_pitch), int(dst_image_rows))

    def crop_nhwc(self, src_bf16, dst_bf16, N, H, W, Cin, pad_h, pad_w, src_row_pitch=0, src_image_rows=0):
        self._call("pcnn_crop_nhwc_bf16", _p(src_bf16), _p(dst_bf16), N, H, W, Cin, int(pad_h), int(pad_w), int(src_row_pitch), int(src_image_rows))

    def softmax_ce(self, logits, labels, B, n, prob=None, d=None, loss=None):
        self._call("pcnn_softmax_ce", _p(logits), _p(labels), int(B), int(n), _p(prob), _p(d), _p(loss))

    def softmax_ce_bf16(self, logits, labels, N, O, scale, dlogits, loss=None, pred=None):
        """pcnn_softmax_ce_bf16: bf16 logits [N][O] and uint8 labels -> dlogits = bf16((softmax - onehot) * scale) (may be logits
        itself), fp32 loss [N] and int32 pred [N] (each None to skip)"""
        self._call("pcnn_softmax_ce_bf16", _p(logits), _p(labels), int(N), int(O), float(scale), _p(dlogits), _p(loss), _p(pred))

    def softmax_ce_soft_bf16(self, logits, labels, N, O, scale, dlogits, loss=None, pred=None, labels_b=None, lam=1.0, smoothing=0.0):
        """pcnn_softmax_ce_soft_bf16: as softmax_ce_bf16 against the fp32 target q = (lam onehot(labels) + (1 - lam)
        onehot(labels_b)) (1 - smoothing) + smoothing / O (labels_b None: onehot(labels)), the target of a MixUp / CutMix batch
        (MixedLabels) with label smoothing"""
        self._call("pcnn_softmax_ce_soft_bf16", _p(logits), _p(labels), _p(labels_b), float(lam), float(smoothing), int(N), int(O),
                   float(scale), _p(dlogits), _p(loss), _p(pred))

    def softmax_ce_pixels_bf16(self, logits, targets, pixels, O, ignore_index, dlogits, count, loss=None, pred=None):
        """pcnn_softmax_ce_pixels_bf16: cross_entropy(ignore_index=ignore_index) with mean reduction over bf16 logits [pixels][O]
        and uint8 targets [pixels].  count (device int32 [1]) receives the non-ignored pixels; every other row gets
        softmax_ce_bf16's row at scale RN32(1 / count); ignored rows get dlogits +0 and loss 0.  ignore_index -1 ignores none."""
        self._call("pcnn_softmax_ce_pixels_bf16", _p(logits), _p(targets), int(pixels), int(O), int(ignore_index), _p(dlogits), _p(loss),
                   _p(pred), _p(count))

    def conv_transpose_fwd(self, x, filt, bias, y, N, H, W, C_in, C_out, R, S, stride=1, padding=(0, 0), output_padding=(0, 0), row_pitch=0,
                           image_rows=0, act=0):
        """pcnn_conv_transpose_fwd: y = act(conv_transpose2d(x, w, bias, stride, padding, output_padding)) with x dense bf16
        [N][H][W][C_in], filt the fp32 master [C_in][R][S][C_out] (torch's weight permuted (0, 2, 3, 1)), bias fp32 [C_out] or None,
        y [N][H_out][W_out][C_out] at row_pitch (0 = W_out C_out) / image_rows (0 = H_out)"""
        ph, pw = (int(v) for v in padding)
        oh, ow = (int(v) for v in output_padding)
        self._call("pcnn_conv_transpose_fwd", _p(x), _p(filt), _p(bias), _p(y), int(N), int(H), int(W), int(C_in), int(C_out), int(R), int(S),
                   int(stride), ph, pw, oh, ow, int(row_pitch or 0), int(image_rows), int(act))

    def upsample_bilinear_fwd(self, x, y, N, H, W, Cin, H_out, W_out):
        """pcnn_upsample_bilinear_nhwc_bf16_fwd: interpolate(size=(H_out, W_out), mode="bilinear", align_corners=False) of dense
        bf16 [N][H][W][C] into dense y [N][H_out][W_out][C]"""
        self._call("pcnn_upsample_bilinear_nhwc_bf16_fwd", _p(x), _p(y), int(N), int(H), int(W), int(Cin), int(H_out), int(W_out))

    def upsample_bilinear_bwd(self, dy, dx, N, H, W, Cin, H_out, W_out):
        """pcnn_upsample_bilinear_nhwc_bf16_bwd: the gradient of that resize, gathered in a fixed order (no atomics), every dx element
        written"""
        self._call("pcnn_upsample_bilinear_nhwc_bf16_bwd", _p(dy), _p(dx), int(N), int(H), int(W), int(Cin), int(H_out), int(W_out))

    def pixel_shuffle(self, x, y, N, H, W, Cin, r):
        """pcnn_pixel_shuffle_nhwc_bf16: F.pixel_shuffle(x, r) on dense bf16 NHWC, x [N][H][W][C r^2] -> y [N][H r][W r][C],
        y[n][h r + i][w r + j][c] = x[n][h][w][c r^2 + i r + j], every element a bit copy"""
        self._call("pcnn_pixel_shuffle_nhwc_bf16", _p(x), _p(y), int(N), int(H), int(W), int(Cin), int(r))

    def pixel_unshuffle(self, x, y, N, H, W, Cin, r):
        """pcnn_pixel_unshuffle_nhwc_bf16: F.pixel_unshuffle(x, r) on dense bf16 NHWC, x [N][H][W][C] -> y [N][H / r][W / r][C r^2],
        the inverse of pixel_shuffle (and its backward)"""
        self._call("pcnn_pixel_unshuffle_nhwc_bf16", _p(x), _p(y), int(N), int(H), int(W), int(Cin), int(r))

    def regression_loss_bf16(self, pred, target, pixels, C, dpred, loss=None, mode=LOSS_MSE, target_stride=None, scale=None):
        """pcnn_regression_loss_bf16: mse_loss (mode LOSS_MSE) or l1_loss (LOSS_L1) of bf16 pred [pixels][C] against the first C
        channels of bf16 target [pixels][target_stride] (None = C).  dpred (may be pred) receives the gradient at scale (None =
        1 / (pixels C), the gradient of reduction="mean"); loss (fp32 [pixels] or None) the unscaled sum of each pixel's terms."""
        ts = int(C) if target_stride is None else int(target_stride)
        if scale is None:
            n = int(pixels) * int(C)
            scale = 1.0 / n if n > 0 else 1.0             # n <= 0: a shape the call refuses
        self._call("pcnn_regression_loss_bf16", _p(pred), _p(target), ts, int(pixels), int(C), int(mode), float(scale), _p(dpred),
                   _p(loss))

    def bce_logits_loss_bf16(self, logits, target, pixels, C, dlogits, loss=None, target_stride=None, scale=None):
        """pcnn_bce_logits_bf16: binary_cross_entropy_with_logits of bf16 logits [pixels][C] against the first C channels of bf16
        probabilities target [pixels][target_stride] (None = C).  dlogits (may be logits) receives scale (sigmoid(x) - t), scale None =
        1 / (pixels C), the gradient of reduction="mean"; loss (fp32 [pixels] or None) the unscaled sum of each pixel's terms."""
        ts = int(C) if target_stride is None else int(target_stride)
        if scale is None:
            n = int(pixels) * int(C)
            scale = 1.0 / n if n > 0 else 1.0             # n <= 0: a shape the call refuses
        self._call("pcnn_bce_logits_bf16", _p(logits), _p(target), ts, int(pixels), int(C), float(scale), _p(dlogits), _p(loss))

    def gaussian_latent_fwd(self, stats, z, R, L, seed, call, kl=None, training=True, ld=None, ldz=None):
        """pcnn_gaussian_latent_bf16_fwd: z [R][ldz] = mu + exp(lv / 2) eps (training) or mu (eval) from stats [R][ld] (mu in
        columns 0 .. L-1, lv in L .. 2L-1; ld None = 2L, ldz None = L), eps the Philox normals of (seed, call); kl (fp32 [R] or
        None) each row's KL divergence from N(0, I).  z may be stats when ldz == ld."""
        ld = 2 * int(L) if ld is None else int(ld)
        ldz = int(L) if ldz is None else int(ldz)
        self._call("pcnn_gaussian_latent_bf16_fwd", _p(stats), ld, _p(z), ldz, _p(kl), int(R), int(L), int(seed), int(call),
                   int(bool(training)))

    def gaussian_latent_bwd(self, stats, dz, dstats, R, L, seed, call, kl_scale, ld=None, ldz=None):
        """pcnn_gaussian_latent_bf16_bwd: dstats [R][ld] (may be stats) = (dz + kl_scale mu, dz eps exp(lv / 2) / 2 + kl_scale
        (exp(lv) - 1) / 2), eps drawn again from the training forward's (seed, call); kl_scale weighs the KL term (beta / N for
        the batch mean)."""
        ld = 2 * int(L) if ld is None else int(ld)
        ldz = int(L) if ldz is None else int(ldz)
        self._call("pcnn_gaussian_latent_bf16_bwd", _p(stats), ld, _p(dz), ldz, _p(dstats), int(R), int(L), int(seed), int(call),
                   float(kl_scale))

    def augment_mask(self, masks, n, H, W, first, N, masks_out, shuffle=1, pad=0, flip=0, seed=0, epoch=0, mask_fill=255):
        """pcnn_augment_mask_u8: the uint8 masks [n][H][W] of augment's batch with the same arguments, each permuted, cropped and
        flipped exactly as its image, the padding filled with mask_fill, into masks_out [N][H][W]"""
        self._call("pcnn_augment_mask_u8", _p(masks), int(n), int(H), int(W), int(first), int(N), int(shuffle), int(pad), int(flip), int(seed),
                   int(epoch), int(mask_fill), _p(masks_out))

    def linear_wgrad(self, plan, x, dy, dw):
        """pcnn_linear_wgrad: dW fp32 [O][P][Q][C] = dy^T x, the shape from the LinearPlan"""
        self._call("pcnn_linear_wgrad", plan.plan, _p(x), _p(dy), _p(dw))

    def linear_dgrad(self, plan, dy, dx):
        """pcnn_linear_dgrad: dx = dy W with the plan's bf16 weights, written in x's layout (pad untouched)"""
        self._call("pcnn_linear_dgrad", plan.plan, _p(dy), _p(dx))

    def dwconv_wgrad(self, plan, x, dy, dw):
        """pcnn_dwconv_wgrad: dw fp32 [C][R][S] = the sum over the pixels of dy * x (x +0 outside the image), overwritten; the shape
        from the DepthwiseConvPlan"""
        self._call("pcnn_dwconv_wgrad", plan.plan, _p(x), _p(dy), _p(dw))

    def dwconv_dgrad(self, plan, dy, dx):
        """pcnn_dwconv_dgrad: dx dense bf16 [N][H][W][C] from dy with the plan's bf16 filters, every element written"""
        self._call("pcnn_dwconv_dgrad", plan.plan, _p(dy), _p(dx))

    def gconv_wgrad(self, plan, x, dy, dw):
        """pcnn_gconv_wgrad: dw fp32 [K][R][S][Cg] = the sum over the pixels of dy * x of the filter's group (x +0 outside the image),
        overwritten; the shape from the GroupedConvPlan"""
        self._call("pcnn_gconv_wgrad", plan.plan, _p(x), _p(dy), _p(dw))

    def gconv_dgrad(self, plan, dy, dx):
        """pcnn_gconv_dgrad: dx dense bf16 [N][H][W][C] from dy with the plan's bf16 filters, every element written"""
        self._call("pcnn_gconv_dgrad", plan.plan, _p(dy), _p(dx))

    def se_scale_fwd(self, x, s, y, N, H, W, Cin, r=None, act=0):
        """pcnn_se_scale_nhwc_bf16_fwd: y = bf16(act(x * s[n][c] (+ r))) over dense bf16 [N][H][W][C], s dense bf16 [N][C] (a
        LinearLayer's y with O = C); act ACT_NONE or ACT_RELU"""
        self._call("pcnn_se_scale_nhwc_bf16_fwd", _p(x), _p(s), _p(r), _p(y), int(N), int(H), int(W), int(Cin), int(act))

    def se_scale_bwd_gate(self, x, y, dy, g, ds, N, H, W, Cin, dy2=None, act=0):
        """pcnn_se_scale_nhwc_bf16_bwd_gate: g = bf16(act'(dy (+ dy2))) (may be dy itself; the gradient of the forward's r) and
        ds[n][c] = bf16 of the sum over the pixels of g * x in GAP's order, the dy of the linear layer that wrote s; y (the forward's
        output) is read at ACT_RELU only"""
        self._call("pcnn_se_scale_nhwc_bf16_bwd_gate", _p(x), _p(y), _p(dy), _p(dy2), _p(g), _p(ds), int(N), int(H), int(W), int(Cin),
                   int(act))

    def se_scale_bwd_input(self, g, s, dx, N, H, W, Cin, dpool=None, dpool_row_pitch=None):
        """pcnn_se_scale_nhwc_bf16_bwd_input: dx = bf16(g * s[n][c] (+ dpool[n][c] / (H*W))), every element written (dx may be g);
        dpool [N][dpool_row_pitch] is the squeeze branch's gradient at the pooled x (row pitch None = C rounded up to 8)"""
        self._call("pcnn_se_scale_nhwc_bf16_bwd_input", _p(g), _p(s), _p(dpool), int(dpool_row_pitch or 0), _p(dx), int(N), int(H), int(W),
                   int(Cin))

    def dropout(self, x, y, N, row_elems, p, seed, call, per_sample=False, r=None, row_pitch=None):
        """pcnn_dropout_bf16: y = bf16(x * m (+ r)) over N bf16 rows of row_elems elements, row_pitch apart (None = dense), m = 0 or
        1 / (1 - p) from the Philox draw of (seed, call) at each element (per_sample False) or each row (True).  y may be x or r.
        The backward is the same call on dy with the forward's (p, seed, call, per_sample) and no r."""
        self._call("pcnn_dropout_bf16", _p(x), _p(r), _p(y), int(N), int(row_elems), int(row_pitch or 0), float(p), int(per_sample),
                   int(seed), int(call))

    def augment(self, images, labels, n, H, W, C, first, N, x, labels_out=None, shuffle=1, pad=0, flip=0, seed=0, epoch=0, mean=None,
                std=None, C_out=None, row_pitch=0, image_rows=0):
        """pcnn_augment_u8_bf16: epoch positions first .. first + N - 1 of the uint8 dataset images [n][H][W][C] (labels [n] or None)
        into x [N][image_rows][row_pitch] bf16 with C_out channels (None = C) and labels_out [N]: image pi(e) when shuffle, cropped
        from the image padded by pad with zeros, flipped when flip, then (u / 255 - mean) / std per channel (None = 0 / 1)."""
        Cin = int(C)
        m, s = channel_stats(mean, Cin, "mean"), channel_stats(std, Cin, "std")
        self._call("pcnn_augment_u8_bf16", _p(images), _p(labels), int(n), int(H), int(W), Cin, int(first), int(N), int(shuffle), int(pad),
                   int(flip), int(seed), int(epoch), None if m is None else m.ctypes.data, None if s is None else s.ctypes.data, _p(x),
                   Cin if C_out is None else int(C_out), int(row_pitch or 0), int(image_rows or 0), _p(labels_out))

    def augment_mix(self, images, labels, n, H, W, C, first, N, x, labels_out=None, labels_b_out=None, mode=MIX_MIXUP, lam=1.0,
                    box=(0, 0, 0, 0), shuffle=1, pad=0, flip=0, seed=0, epoch=0, mean=None, std=None, C_out=None, row_pitch=0,
                    image_rows=0):
        """pcnn_augment_mix_u8_bf16: augment's batch with MixUp (mode MIX_MIXUP: lam j + (1 - lam) j' in fp32) or CutMix
        (MIX_CUTMIX: the box (x1, y1, x2, y2) of output pixels from j') of each position j and its partner j' = (j + N - 1) mod N;
        labels_b_out [N] receives the partners' labels"""
        Cin = int(C)
        m, s = channel_stats(mean, Cin, "mean"), channel_stats(std, Cin, "std")
        x1, y1, x2, y2 = (int(v) for v in box)
        self._call("pcnn_augment_mix_u8_bf16", _p(images), _p(labels), int(n), int(H), int(W), Cin, int(first), int(N), int(shuffle),
                   int(pad), int(flip), int(seed), int(epoch), None if m is None else m.ctypes.data, None if s is None else s.ctypes.data,
                   _p(x), Cin if C_out is None else int(C_out), int(row_pitch or 0), int(image_rows or 0), _p(labels_out), int(mode),
                   float(lam), x1, y1, x2, y2, _p(labels_b_out))

    def augment_resized(self, images, labels, n, H, W, C, first, N, x, H_out, W_out, labels_out=None, mode=RESIZE_TRAIN,
                        scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3), resize_size=0, shuffle=1, flip=0, seed=0, epoch=0, mean=None, std=None,
                        C_out=None, row_pitch=0, image_rows=0):
        """pcnn_augment_resized_u8_bf16: augment's batch at H_out x W_out pixels per image.  mode RESIZE_TRAIN:
        RandomResizedCrop((H_out, W_out), scale, ratio, antialias=True), then the flip when flip; RESIZE_EVAL: Resize(resize_size)
        + CenterCrop((H_out, W_out)).  Both resample as torch's uint8 bilinear antialiased resize, then (u / 255 - mean) / std."""
        Cin = int(C)
        m, s = channel_stats(mean, Cin, "mean"), channel_stats(std, Cin, "std")
        self._call("pcnn_augment_resized_u8_bf16", _p(images), _p(labels), int(n), int(H), int(W), Cin, int(first), int(N), int(shuffle),
                   int(flip), int(seed), int(epoch), None if m is None else m.ctypes.data, None if s is None else s.ctypes.data, _p(x),
                   int(H_out), int(W_out), Cin if C_out is None else int(C_out), int(row_pitch or 0), int(image_rows or 0), _p(labels_out),
                   int(mode), float(scale[0]), float(scale[1]), float(ratio[0]), float(ratio[1]), int(resize_size or 0))

    def augment_trivial(self, images, labels, n, H, W, C, first, N, x, workspace, labels_out=None, trivial=TRIVIAL_NEAREST,
                        erase_p=0.0, erase_scale=(0.02, 0.33), erase_ratio=(0.3, 3.3), crop_size=None, scale=(0.08, 1.0),
                        ratio=(3 / 4, 4 / 3), shuffle=1, pad=0, flip=0, seed=0, epoch=0, mean=None, std=None, C_out=None, row_pitch=0,
                        image_rows=0):
        """pcnn_augment_trivial_u8_bf16: a training batch of augment's crop, pad and flip (crop_size None) or augment_resized's
        RandomResizedCrop(crop_size, scale, ratio) and flip, then TrivialAugmentWide (trivial TRIVIAL_NEAREST / TRIVIAL_BILINEAR, or
        TRIVIAL_NONE), (u / 255 - mean) / std, and RandomErasing(erase_p, erase_scale, erase_ratio, value=0).  workspace is a device
        buffer of at least augment_trivial_info(...)["ws_bytes"] bytes that holds the uint8 crops between the two launches."""
        Cin = int(C)
        m, s = channel_stats(mean, Cin, "mean"), channel_stats(std, Cin, "std")
        hw = (0, 0) if crop_size is None else tuple(int(v) for v in crop_size)
        self._call("pcnn_augment_trivial_u8_bf16", _p(images), _p(labels), int(n), int(H), int(W), Cin, int(first), int(N), int(shuffle),
                   int(pad), int(flip), int(seed), int(epoch), None if m is None else m.ctypes.data, None if s is None else s.ctypes.data,
                   _p(x), Cin if C_out is None else int(C_out), int(row_pitch or 0), int(image_rows or 0), _p(labels_out),
                   int(crop_size is not None), *hw, float(scale[0]), float(scale[1]), float(ratio[0]), float(ratio[1]), int(trivial),
                   float(erase_p), float(erase_scale[0]), float(erase_scale[1]), float(erase_ratio[0]), float(erase_ratio[1]),
                   _p(workspace), 0 if workspace is None else int(workspace.nbytes))


class MixedLabels(NamedTuple):
    """The targets of a mixed training batch: image j is lam parts labels[j] and 1 - lam parts labels_b[j] (lam_adjusted, the
    box's complement over the image, for CutMix).  kind is "mixup" or "cutmix"; box (x1, y1, x2, y2) the CutMix box, else None."""
    labels: object
    labels_b: object
    lam: float
    kind: str
    box: Optional[tuple]


def mix_draws(seed, epoch, step, H, W, mixup_alpha, cutmix_alpha):
    """(kind, lam, box, lam_adjusted) of training batch `step` of `epoch` (box and lam_adjusted None for MixUp), drawn from numpy's
    Philox generator keyed by seed with counter (0, 0, epoch, step), so a function of (seed, epoch, step) alone.  In order:
      1. with both alphas > 0, u = random(): CutMix iff u < 1/2 (torchvision's RandomChoice([MixUp, CutMix])); otherwise the kind
         whose alpha is > 0;
      2. lam = beta(alpha, alpha) with that kind's alpha;
      3. CutMix: r_x = integers(W), then r_y = integers(H), and the box and lam_adjusted exactly as v2.CutMix.make_params forms
         them (double arithmetic, int() truncation, clamping to the image).
    numpy does not promise the same Generator.beta stream across numpy versions, so a different numpy may draw other batches."""
    rng = np.random.Generator(np.random.Philox(key=int(seed), counter=np.array([0, 0, int(epoch), int(step)], np.uint64)))
    cutmix = rng.random() < 0.5 if (mixup_alpha > 0 and cutmix_alpha > 0) else cutmix_alpha > 0
    alpha = cutmix_alpha if cutmix else mixup_alpha
    lam = float(rng.beta(alpha, alpha))
    if not cutmix:
        return "mixup", lam, None, None
    r_x, r_y = int(rng.integers(W)), int(rng.integers(H))
    r = 0.5 * math.sqrt(1.0 - lam)
    r_w_half, r_h_half = int(r * W), int(r * H)
    x1, y1 = max(r_x - r_w_half, 0), max(r_y - r_h_half, 0)
    x2, y2 = min(r_x + r_w_half, W), min(r_y + r_h_half, H)
    return "cutmix", lam, (x1, y1, x2, y2), float(1.0 - (x2 - x1) * (y2 - y1) / (W * H))


class ConvPlan:
    """bf16 tensor-core convolution plan (pcnn_conv_tc_*): filters fp32 KRSC on the host, activations NHWC bf16.  act is
    ACT_NONE (0), ACT_SIGMOID (1) or ACT_RELU (3), fused after the bias; any other value is refused."""

    def __init__(self, engine, N, H, W, C, K, R, S, filt, bias=None, act=0, row_pitch=None, image_rows=0, stride=1):
        self.shape = (N, H, W, C, K, R, S)
        self.row_pitch = int(row_pitch if row_pitch is not None else (W * C + 7) // 8 * 8)
        self._create(engine, "pcnn_conv_tc_plan_create_strided", filt, K * R * S * C, bias,
                     N, H, W, C, K, R, S, int(stride), self.row_pitch, int(image_rows), int(act))
        self.out_shape = (N, (H - R) // stride + 1, (W - S) // stride + 1, K)

    def _create(self, engine, fn, filt, nf, bias, *args):
        """self.plan from the create call fn(ctx, *args, filters, bias, &plan): filt (nf elements) and bias (or None) as fp32"""
        self.engine = engine
        filt = np.ascontiguousarray(filt, np.float32)
        assert filt.size == nf
        b = None if bias is None else np.ascontiguousarray(bias, np.float32)
        plan = C_.c_void_p()
        check(fn, getattr(lib(), fn)(engine.ctx, *args, filt.ctypes.data, None if b is None else b.ctypes.data, C_.byref(plan)))
        self.plan = plan

    def fwd(self, x_bf16_dev, y_bf16_dev):
        check("pcnn_conv_tc_fwd", lib().pcnn_conv_tc_fwd(self.engine.ctx, self.plan, _p(x_bf16_dev), _p(y_bf16_dev)))

    def set_params(self, filt_dev, bias_dev=None):
        """new filters (fp32 KRSC) and / or bias (fp32 [K]) from device memory, enqueued on the engine's stream
        (pcnn_conv_plan_set_params); None leaves that part unchanged"""
        check("pcnn_conv_plan_set_params", lib().pcnn_conv_plan_set_params(self.engine.ctx, self.plan, _p(filt_dev), _p(bias_dev)))

    def close(self):
        if self.plan and self.engine.ctx:
            lib().pcnn_conv_tc_plan_destroy(self.engine.ctx, self.plan)
        self.plan = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class WideConvPlan(ConvPlan):
    """The wide-channel forward (pcnn_conv_wide_plan_create): the shapes ConvPlan refuses, C % 8 == 0, K % 8 == 0, K <= 256.
    padding=(pad_h, pad_w) other than (0, 0) zero-pads x as conv2d(padding=...) does (pcnn_conv_wide_plan_create_padded);
    dilation=(dil_h, dil_w) other than (1, 1) spaces the taps as conv2d(dilation=...) does (pcnn_conv_wide_plan_create_dilated).
    Run and closed like ConvPlan."""

    def __init__(self, engine, N, H, W, C, K, R, S, filt, bias=None, act=0, row_pitch=None, image_rows=0, stride=1, padding=(0, 0),
                 dilation=(1, 1)):
        self.shape = (N, H, W, C, K, R, S)
        self.row_pitch = int(row_pitch if row_pitch is not None else (W * C + 7) // 8 * 8)
        ph, pw = (int(v) for v in padding)
        dh, dw = (int(v) for v in dilation)
        if (dh, dw) != (1, 1):
            fn, extra = "pcnn_conv_wide_plan_create_dilated", (ph, pw, dh, dw)
        elif (ph, pw) != (0, 0):
            fn, extra = "pcnn_conv_wide_plan_create_padded", (ph, pw)
        else:
            fn, extra = "pcnn_conv_wide_plan_create", ()
        self._create(engine, fn, filt, K * R * S * C, bias, N, H, W, C, K, R, S, int(stride), *extra, self.row_pitch, int(image_rows), int(act))
        self.out_shape = (N, (H + 2 * ph - dh * (R - 1) - 1) // stride + 1, (W + 2 * pw - dw * (S - 1) - 1) // stride + 1, K)


class LinearPlan(ConvPlan):
    """A fully connected layer's plan (pcnn_linear_plan_create): x [N][image_rows][row_pitch] bf16 holding P x Q pixels of C
    channels per image, w fp32 [O][P][Q][C], y dense bf16 [N][O], 1 <= O <= 256.  row_pitch None or 0 = Q*C rounded up to 8.  Run,
    refreshed and closed like ConvPlan; its gradients are Engine.linear_wgrad / linear_dgrad."""

    def __init__(self, engine, N, P, Q, C, O, w, bias=None, act=0, row_pitch=None, image_rows=0):
        self.shape = (N, P, Q, C, O)
        self.row_pitch = int(row_pitch or (Q * C + 7) // 8 * 8)
        self._create(engine, "pcnn_linear_plan_create", w, O * P * Q * C, bias, N, P, Q, C, O, self.row_pitch, int(image_rows), int(act))
        self.out_shape = (N, O)


class DepthwiseConvPlan(ConvPlan):
    """A depthwise convolution's plan (pcnn_dwconv_plan_create): conv2d(x, w, b, stride, padding, groups=C) with x dense bf16
    [N][H][W][C], y dense bf16 [N][P][Q][C], filters fp32 [C][R][S] (torch's weight [C][1][R][S] reshaped), bias fp32 [C].  act
    ACT_NONE (0) or ACT_RELU (3).  dilation=(dil_h, dil_w) other than (1, 1) is conv2d(dilation=...)
    (pcnn_dwconv_plan_create_dilated).  Run, refreshed and closed like ConvPlan; its gradients are Engine.dwconv_wgrad / dwconv_dgrad."""

    def __init__(self, engine, N, H, W, C, R, S, filt, bias=None, act=0, stride=1, padding=(0, 0), dilation=(1, 1)):
        self.shape = (N, H, W, C, R, S)
        ph, pw = (int(v) for v in padding)
        dh, dw = (int(v) for v in dilation)
        if (dh, dw) != (1, 1):
            self._create(engine, "pcnn_dwconv_plan_create_dilated", filt, C * R * S, bias, N, H, W, C, R, S, int(stride), ph, pw, dh, dw,
                         int(act))
        else:
            self._create(engine, "pcnn_dwconv_plan_create", filt, C * R * S, bias, N, H, W, C, R, S, int(stride), ph, pw, int(act))
        self.out_shape = (N, (H + 2 * ph - dh * (R - 1) - 1) // stride + 1, (W + 2 * pw - dw * (S - 1) - 1) // stride + 1, C)


class GroupedConvPlan(ConvPlan):
    """A grouped convolution's plan (pcnn_gconv_plan_create): conv2d(x, w, b, stride, padding, groups=G) with x dense bf16
    [N][H][W][C], y dense bf16 [N][P][Q][K], filters fp32 [K][R][S][Cg] (torch's weight [K][Cg][R][S] permuted), bias fp32 [K].  act
    ACT_NONE (0) or ACT_RELU (3).  Run, refreshed and closed like ConvPlan; its gradients are Engine.gconv_wgrad / gconv_dgrad."""

    def __init__(self, engine, N, H, W, C, K, G, R, S, filt, bias=None, act=0, stride=1, padding=(0, 0)):
        self.shape = (N, H, W, C, K, G, R, S)
        ph, pw = (int(v) for v in padding)
        assert G >= 1
        self._create(engine, "pcnn_gconv_plan_create", filt, K * R * S * (C // G), bias, N, H, W, C, K, G, R, S, int(stride), ph, pw,
                     int(act))
        self.out_shape = (N, (H + 2 * ph - R) // stride + 1, (W + 2 * pw - S) // stride + 1, K)


class _PlanLayer:
    """What the plan-backed layers share: fp32 master filters and bias, their gradients dw and db, all in DeviceArrays, and a plan
    holding the filters in bf16.  A subclass builds its plan, calls _own(engine, plan, filt, bias) with the host masters in the
    plan's element order, and supplies _grads(dy, dx): the weight gradient into dw and, when dx is given, the input gradient."""

    def _own(self, engine, plan, filt, bias):
        self.engine, self.plan = engine, plan
        self.out_shape = plan.out_shape
        self.pixels = int(np.prod(self.out_shape[:-1]))
        self.filt = DeviceArray.from_host(engine, filt)
        self.bias = None if bias is None else DeviceArray.from_host(engine, bias)
        self.dw = engine.array(filt.shape)
        self.db = None if bias is None else engine.array(bias.size)
        self._x = None

    def forward(self, x, y):
        """y = act(layer(x) + bias) with the plan's bf16 filters.  The layer keeps x: backward's weight gradient reads it."""
        self.plan.fwd(x, y)
        self._x = x

    def backward(self, y, dy, dx=None):
        """Gradients of the most recent forward, whose output y was: dw, db (with a bias) and dx (when given; a first layer
        passes None).  dy is CONSUMED: with a sigmoid or a ReLU it is overwritten in place by the gradient at the pre-activation,
        which the weight and input gradients then read (pcnn_conv_bias_act_bwd over the output's pixels, skipped without
        activation and bias)."""
        if self.act or self.bias is not None:
            self.engine.conv_bias_act_bwd(y if self.act else None, dy, dy if self.act else None, self.db, self.pixels, self.out_shape[-1],
                                          self.act)
        self._grads(dy, dx)

    def sgd(self, lr):
        """w += (-lr) * dw and b += (-lr) * db in fp32 on the masters, then the plan refreshed from them, all on the engine's stream"""
        self.engine.apply_grad_scaled(self.filt, self.dw, int(np.prod(self.filt.shape)), -lr)
        if self.bias is not None:
            self.engine.apply_grad_scaled(self.bias, self.db, self.out_shape[-1], -lr)
        self.plan.set_params(self.filt, self.bias)

    def optim_tensors(self):
        """(param, grad, plan, plan part, is norm or bias) of each trainable tensor: the table SGD and AdamW are built from"""
        return [(self.filt, self.dw, self.plan, 1, False)] + ([] if self.bias is None else [(self.bias, self.db, self.plan, 2, True)])

    def params(self):
        """host copies (filters in the plan's element order, bias or None) of the fp32 masters"""
        return self.filt.to_host(), None if self.bias is None else self.bias.to_host()

    def close(self):
        self.plan.close()
        for a in (self.filt, self.bias, self.dw, self.db):
            if a is not None:
                a.free()


class ConvLayer(_PlanLayer):
    """One bf16 convolution layer trained on the device: forward, backward and an SGD step with no host round trip.

    It owns fp32 master filters (KRSC) and bias, their gradients dw and db, all in DeviceArrays, and a forward plan of the family
    that serves the shape (conv_layer_family: the row-Toeplitz plan for few channels without padding, the wide plan otherwise).
    Activations are NHWC bf16: x with row_pitch (None = W*C rounded up to 8) and image_rows (0 = H), y and dy dense
    [N][P][Q][K], dx in x's layout.  act ACT_SIGMOID (1) is a sigmoid after the bias, ACT_RELU (3) a ReLU, ACT_NONE (0) none.
    dilation=(dil_h, dil_w) spaces the taps as conv2d(dilation=...); a dilated layer is always the wide plan's (C % 8 == 0)."""

    def __init__(self, engine, N, H, W, C, K, R, S, filt, bias=None, act=0, stride=1, padding=(0, 0), row_pitch=None, image_rows=0,
                 dilation=(1, 1)):
        self.shape = (N, H, W, C, K, R, S)
        self.act, self.stride = int(act), int(stride)
        self.padding = tuple(int(v) for v in padding)
        self.dilation = tuple(int(v) for v in dilation)
        self.row_pitch = int(row_pitch if row_pitch is not None else (W * C + 7) // 8 * 8)
        self.image_rows = int(image_rows)
        self.family = conv_layer_family(N, H, W, C, K, R, S, self.stride, self.padding, self.row_pitch, self.image_rows, self.dilation)
        filt = np.ascontiguousarray(filt, np.float32).reshape(K, R, S, C)
        bias = None if bias is None else np.ascontiguousarray(bias, np.float32).reshape(K)
        if self.family == "narrow":
            plan = ConvPlan(engine, N, H, W, C, K, R, S, filt, bias, act=act, row_pitch=self.row_pitch, image_rows=self.image_rows,
                            stride=self.stride)
        else:
            plan = WideConvPlan(engine, N, H, W, C, K, R, S, filt, bias, act=act, row_pitch=self.row_pitch, image_rows=self.image_rows,
                                stride=self.stride, padding=self.padding, dilation=self.dilation)
        self._own(engine, plan, filt, bias)

    def _grads(self, dy, dx):
        N, H, W, C, K, R, S = self.shape
        e = self.engine
        if self.family == "narrow":
            e.conv_wgrad(self._x, dy, self.dw, N, H, W, C, K, R, S, self.row_pitch, self.image_rows, self.stride)
            if dx is not None:
                e.conv_dgrad(dy, self.filt, dx, N, H, W, C, K, R, S, self.row_pitch, self.image_rows, self.stride)
        else:
            e.conv_wide_wgrad(self._x, dy, self.dw, N, H, W, C, K, R, S, self.row_pitch, self.image_rows, self.stride, self.padding,
                              self.dilation)
            if dx is not None:
                e.conv_wide_dgrad(dy, self.filt, dx, N, H, W, C, K, R, S, self.row_pitch, self.image_rows, self.stride, self.padding,
                                  self.dilation)


class ConvTransposeLayer(_PlanLayer):
    """A transposed convolution trained on the device, as torch.nn.ConvTranspose2d(C_in, C_out, (R, S), stride, padding,
    output_padding) with groups 1 and dilation 1:  H_out = (H - 1) stride - 2 pad_h + R + output_padding_h, W_out the same.
    weight has torch's layout [C_in][C_out][R][S]; the fp32 master `filt` is held as the adjoint convolution's KRSC [C_in][R][S][C_out]
    (K = C_in filters over C = C_out channels), torch's weight permuted (0, 2, 3, 1).  x is dense bf16 [N][H][W][C_in]; y and dy are
    [N][H_out][W_out][C_out] at row_pitch (None = dense) and image_rows (0 = H_out); dx is dense like x.
      forward:  pcnn_conv_transpose_fwd (the wide input gradient with a bias and activation epilogue), from the master on every call;
      backward: pcnn_conv_bias_act_bwd over y (with a bias or an activation), dx = the forward of the adjoint convolution's
                WideConvPlan on dy, dw = its weight gradient with the activations swapped (x = dy, dy = x).
    The adjoint plan holds the master's bf16 rounding for dx and is what the optimizers refresh, so call backward before sgd or an
    optimizer step.  With a bias or an activation y must be dense (pcnn_conv_bias_act_bwd reads it so) and C_out <= 256."""

    def __init__(self, engine, N, H, W, C_in, C_out, R, S, weight, bias=None, act=0, stride=1, padding=(0, 0), output_padding=(0, 0),
                 row_pitch=None, image_rows=0):
        self.act, self.stride = int(act), int(stride)
        self.padding = tuple(int(v) for v in padding)
        self.output_padding = tuple(int(v) for v in output_padding)
        self.info = conv_transpose_info(N, H, W, C_in, C_out, R, S, self.stride, self.padding, self.output_padding, row_pitch, image_rows,
                                        bias is not None, self.act)
        H_out, W_out = self.info["H_out"], self.info["W_out"]
        self.row_pitch, self.image_rows = self.info["row_pitch"], self.info["image_rows"]
        if (self.act or bias is not None) and (self.row_pitch != W_out * C_out or self.image_rows != H_out):
            raise PcnnError("ConvTransposeLayer", -1, f"row_pitch {self.row_pitch}, image_rows {self.image_rows} with a bias or an activation: "
                            "y must be dense (row_pitch W_out C_out, image_rows H_out), as pcnn_conv_bias_act_bwd reads it")
        self.shape = (N, H, W, C_in, C_out, R, S)
        filt = np.ascontiguousarray(np.asarray(weight, np.float32).reshape(C_in, C_out, R, S).transpose(0, 2, 3, 1))
        bias = None if bias is None else np.ascontiguousarray(bias, np.float32).reshape(C_out)
        plan = WideConvPlan(engine, N, H_out, W_out, C_out, C_in, R, S, filt, None, act=0, row_pitch=self.row_pitch,
                            image_rows=self.image_rows, stride=self.stride, padding=self.padding)
        self._own(engine, plan, filt, bias)
        self.out_shape = (N, H_out, W_out, C_out)
        self.pixels = N * H_out * W_out

    def forward(self, x, y):
        """y = act(conv_transpose2d(x) + bias) from the master's bf16 rounding.  The layer keeps x: backward's weight gradient reads it."""
        N, H, W, C_in, C_out, R, S = self.shape
        self.engine.conv_transpose_fwd(x, self.filt, self.bias, y, N, H, W, C_in, C_out, R, S, self.stride, self.padding, self.output_padding,
                                       self.row_pitch, self.image_rows, self.act)
        self._x = x

    def _grads(self, dy, dx):
        N, H, W, C_in, C_out, R, S = self.shape
        _, H_out, W_out, _ = self.out_shape
        self.engine.conv_wide_wgrad(dy, self._x, self.dw, N, H_out, W_out, C_out, C_in, R, S, self.row_pitch, self.image_rows, self.stride,
                                    self.padding)
        if dx is not None:
            self.plan.fwd(dy, dx)

    def sgd(self, lr):
        """w += (-lr) * dw and b += (-lr) * db in fp32 on the masters, then the adjoint plan refreshed from the filters"""
        self.engine.apply_grad_scaled(self.filt, self.dw, int(np.prod(self.filt.shape)), -lr)
        if self.bias is not None:
            self.engine.apply_grad_scaled(self.bias, self.db, self.out_shape[-1], -lr)
        self.plan.set_params(self.filt)

    def optim_tensors(self):
        """the filters refresh the adjoint plan (part 1); the bias belongs to no plan, the forward reads the master"""
        return [(self.filt, self.dw, self.plan, 1, False)] + ([] if self.bias is None else [(self.bias, self.db, None, 0, True)])

    def weight(self):
        """a host copy of the master in torch's layout [C_in][C_out][R][S]"""
        return self.filt.to_host().reshape(self.filt.shape).transpose(0, 3, 1, 2).copy()


class UpsampleBilinearLayer:
    """Bilinear resizing between two layers (pcnn_upsample_bilinear_nhwc_bf16_fwd / _bwd), as interpolate(size=(H_out, W_out),
    mode="bilinear", align_corners=False): up- or downsampling, without antialiasing.  x and dx are dense bf16 [N][H][W][C], y and
    dy dense [N][H_out][W_out][C].  It keeps no state; info is its partition (upsample_bilinear_info).  The backward gathers each dx
    element in a fixed order, so reruns give the same bits."""

    def __init__(self, engine, N, H, W, C, H_out, W_out):
        self.engine = engine
        self.shape = (int(N), int(H), int(W), int(C), int(H_out), int(W_out))
        self.info = upsample_bilinear_info(*self.shape)
        self.out_shape = (int(N), int(H_out), int(W_out), int(C))

    def forward(self, x, y):
        self.engine.upsample_bilinear_fwd(x, y, *self.shape)

    def backward(self, dy, dx):
        self.engine.upsample_bilinear_bwd(dy, dx, *self.shape)

    def close(self):
        pass


class PixelShuffleLayer:
    """Sub-pixel upsampling between two layers (pcnn_pixel_shuffle_nhwc_bf16), as F.pixel_shuffle(x, r): x and dx dense bf16
    [N][H][W][C r^2] (a convolution's or a per-pixel LinearLayer's output with C r^2 channels), y and dy dense [N][H r][W r][C].  It
    keeps no state; info is its partition (pixel_shuffle_info).  The backward is the unshuffle of dy: a bit copy, like the forward."""

    def __init__(self, engine, N, H, W, C, r):
        self.engine = engine
        self.shape = (int(N), int(H), int(W), int(C), int(r))
        self.info = pixel_shuffle_info(*self.shape)
        pixel_shuffle_info(N, H * r, W * r, C, r, unshuffle=True)      # the backward's shape, refused here rather than mid-step
        self.out_shape = (int(N), int(H) * int(r), int(W) * int(r), int(C))

    def forward(self, x, y):
        self.engine.pixel_shuffle(x, y, *self.shape)

    def backward(self, dy, dx):
        N, H, W, C, r = self.shape
        self.engine.pixel_unshuffle(dy, dx, N, H * r, W * r, C, r)

    def close(self):
        pass


class PixelUnshuffleLayer:
    """Lossless downsampling between two layers (pcnn_pixel_unshuffle_nhwc_bf16), as F.pixel_unshuffle(x, r): x and dx dense bf16
    [N][H][W][C] with H and W multiples of r, y and dy dense [N][H / r][W / r][C r^2].  It keeps no state; info is its partition
    (pixel_shuffle_info).  The backward is the shuffle of dy."""

    def __init__(self, engine, N, H, W, C, r):
        self.engine = engine
        self.shape = (int(N), int(H), int(W), int(C), int(r))
        self.info = pixel_shuffle_info(*self.shape, unshuffle=True)
        pixel_shuffle_info(N, H // r, W // r, C, r)                    # the backward's shape
        self.out_shape = (int(N), int(H) // int(r), int(W) // int(r), int(C) * int(r) * int(r))

    def forward(self, x, y):
        self.engine.pixel_unshuffle(x, y, *self.shape)

    def backward(self, dy, dx):
        N, H, W, C, r = self.shape
        self.engine.pixel_shuffle(dy, dx, N, H // r, W // r, C, r)

    def close(self):
        pass


class GaussianLatentLayer:
    """The reparameterized latent of a variational autoencoder (pcnn_gaussian_latent_bf16_fwd / _bwd): stats [R][ld] bf16 holds mu in
    columns 0 .. L-1 and the log-variance in L .. 2L-1 (an encoder LinearLayer with O = 2L; ld None = 2L), z [R][ldz] (None = L)
    is mu + exp(lv / 2) eps.  kl (a DeviceArray of R floats) receives each row's KL divergence from N(0, I) at every forward.  It
    has no parameters, so no optim_tensors.

    eps is the Philox draw of (seed, call) at each element, call being incremented by every training forward; `call` is a plain
    attribute, so a checkpoint can save and restore it.  backward replays the eps of the most recent training forward:

        enc.forward(h, stats);  lat.forward(stats, z);  dec.forward(z, y)
        dec.backward(y, dy, dz);  lat.backward(dz, dstats, beta / N);  enc.backward(stats, dstats, dh)

    dstats may be stats itself when the encoder's backward does not read its output (no activation)."""

    def __init__(self, engine, R, L, seed, ld=None, ldz=None):
        self.engine = engine
        self.R, self.L = int(R), int(L)
        self.ld = 2 * self.L if ld is None else int(ld)
        self.ldz = self.L if ldz is None else int(ldz)
        self.info = gaussian_latent_info(self.R, self.L, self.ld, self.ldz)
        self.seed = int(seed)
        self.call = 0
        self.kl = engine.array((self.R,), np.float32)
        self._stats = None

    def forward(self, stats, z, training=True):
        """training: call += 1, then z = mu + exp(lv / 2) eps with this call's draw; eval: z = mu.  kl is written in both."""
        if training:
            self.call += 1
            self._stats = stats
        self.engine.gaussian_latent_fwd(stats, z, self.R, self.L, self.seed, self.call, kl=self.kl, training=training, ld=self.ld,
                                        ldz=self.ldz)

    def backward(self, dz, dstats, kl_scale):
        """dstats = the gradient of (the loss behind dz) + kl_scale sum(kl) with respect to the stats of the most recent training
        forward, which must still hold them; dstats may be that buffer (in place)."""
        if self._stats is None:
            raise PcnnError("GaussianLatentLayer.backward", -1, "no training forward to differentiate")
        self.engine.gaussian_latent_bwd(self._stats, dz, dstats, self.R, self.L, self.seed, self.call, kl_scale, ld=self.ld,
                                        ldz=self.ldz)

    def close(self):
        if self.kl is not None:
            self.kl.free()
            self.kl = None


def psnr(pred, target, data_range=1.0):
    """Host evaluation of an image regression (not a hot path): the mean over images (the first axis) of
    10 log10(data_range^2 / MSE_image), in float64; an image with MSE 0 scores +inf."""
    p, t = np.asarray(pred, np.float64), np.asarray(target, np.float64)
    if p.shape != t.shape:
        raise PcnnError("psnr", -1, f"pred {p.shape} and target {t.shape} differ")
    p, t = p.reshape(len(p), -1), t.reshape(len(t), -1)
    mse = ((p - t) ** 2).mean(1)
    with np.errstate(divide="ignore"):
        return float(np.mean(10.0 * np.log10(float(data_range) ** 2 / mse)))


def segmentation_scores(pred, targets, O, ignore_index=255):
    """Host evaluation of a per-pixel prediction (not a hot path): (confusion, iou, miou).  confusion[t][p] counts the pixels with
    target t < O, t != ignore_index, predicted p (0 <= p < O; other predictions, such as the -1 of a NaN row, count in no column but
    still in their target's row total).  iou[c] = confusion[c][c] / (row total + column total - confusion[c][c]), NaN for a class
    absent from both; miou is the mean over the classes whose IoU is not NaN."""
    t = np.asarray(targets).reshape(-1).astype(np.int64)
    p = np.asarray(pred).reshape(-1).astype(np.int64)
    keep = (t != ignore_index) & (t >= 0) & (t < O)
    t, p = t[keep], p[keep]
    rows = np.bincount(t, minlength=O)
    ok = (p >= 0) & (p < O)
    conf = np.bincount(t[ok] * O + p[ok], minlength=O * O).reshape(O, O)
    tp = np.diag(conf).astype(np.float64)
    union = rows + conf.sum(0) - tp
    with np.errstate(invalid="ignore", divide="ignore"):
        iou = np.where(union > 0, tp / np.maximum(union, 1), np.nan)
    present = ~np.isnan(iou)
    return conf, iou, float(iou[present].mean()) if present.any() else float("nan")


class DepthwiseConvLayer(_PlanLayer):
    """A depthwise convolution trained on the device (groups = C: each channel filtered by its own R x S filter), with ConvLayer's
    interface: fp32 masters filt [C][R][S] and bias [C], their gradients dw and db, and a DepthwiseConvPlan holding the filters in
    bf16.  x and dx are dense bf16 [N][H][W][C], y and dy dense [N][P][Q][C]: what a ConvLayer or a BatchNormLayer writes and reads,
    so an inverted-residual block runs with no copies:

        expand.forward(x, ye);  bn1.forward(ye, ze);  dw.forward(ze, yd);  bn2.forward(yd, zd);  project.forward(zd, yp)
        ...;  bn2.backward(zd, dzd, dyd);  dw.backward(yd, dyd, dze);  bn1.backward(ze, dze, dye)

    act ACT_RELU (3) is a ReLU after the bias, ACT_NONE (0) none; the sigmoid is refused.  With a bias or an activation, backward
    first runs pcnn_conv_bias_act_bwd over dy, which takes at most 256 channels: such a layer needs C <= 256.  Without either
    (the usual case in front of a batch norm) C is unlimited.  dx uses the plan's bf16 filters, so call backward before sgd or an
    optimizer step."""

    def __init__(self, engine, N, H, W, C, R, S, filt, bias=None, act=0, stride=1, padding=(0, 0), dilation=(1, 1)):
        self.shape = (N, H, W, C, R, S)
        self.act, self.stride = int(act), int(stride)
        self.padding = tuple(int(v) for v in padding)
        self.dilation = tuple(int(v) for v in dilation)
        self.info = dwconv_info(N, H, W, C, R, S, self.stride, self.padding, self.dilation)
        filt = np.ascontiguousarray(filt, np.float32).reshape(C, R, S)
        bias = None if bias is None else np.ascontiguousarray(bias, np.float32).reshape(C)
        plan = DepthwiseConvPlan(engine, N, H, W, C, R, S, filt, bias, act=act, stride=self.stride, padding=self.padding,
                                 dilation=self.dilation)
        self._own(engine, plan, filt, bias)

    def _grads(self, dy, dx):
        self.engine.dwconv_wgrad(self.plan, self._x, dy, self.dw)
        if dx is not None:
            self.engine.dwconv_dgrad(self.plan, dy, dx)


class GroupedConvLayer(_PlanLayer):
    """A grouped convolution trained on the device (groups = G: each group of C / G input channels feeds its own K / G filters), with
    ConvLayer's interface: fp32 masters filt [K][R][S][Cg] and bias [K], their gradients dw and db, and a GroupedConvPlan holding the
    filters in bf16.  x and dx are dense bf16 [N][H][W][C], y and dy dense [N][P][Q][K]: what a ConvLayer or a BatchNormLayer writes
    and reads, so a ResNeXt bottleneck runs with no copies:

        reduce.forward(x, yr);  bn1.forward(yr, zr);  grouped.forward(zr, yg);  bn2.forward(yg, zg);  expand.forward(zg, ye)
        ...;  bn2.backward(zg, dzg, dyg);  grouped.backward(yg, dyg, dzr);  bn1.backward(zr, dzr, dyr)

    act ACT_RELU (3) is a ReLU after the bias, ACT_NONE (0) none; the sigmoid is refused.  With a bias or an activation, backward
    first runs pcnn_conv_bias_act_bwd over dy, which takes at most 256 channels: such a layer needs K <= 256 and is refused
    otherwise.  Without either (the usual case in front of a batch norm) C and K are unlimited.  dx uses the plan's bf16 filters, so
    call backward before sgd or an optimizer step."""

    def __init__(self, engine, N, H, W, C, K, G, R, S, filt, bias=None, act=0, stride=1, padding=(0, 0)):
        if (int(act) or bias is not None) and K > 256:
            raise PcnnError("GroupedConvLayer", -1, f"K = {K} with a bias or an activation: the bias / activation backward "
                            "(pcnn_conv_bias_act_bwd) takes K <= 256; put a BatchNormLayer after a layer with no bias and act 0")
        self.shape = (N, H, W, C, K, G, R, S)
        self.act, self.stride = int(act), int(stride)
        self.padding = tuple(int(v) for v in padding)
        self.info = gconv_info(N, H, W, C, K, G, R, S, self.stride, self.padding)
        Cg = self.info["Cg"]
        filt = np.ascontiguousarray(filt, np.float32).reshape(K, R, S, Cg)
        bias = None if bias is None else np.ascontiguousarray(bias, np.float32).reshape(K)
        plan = GroupedConvPlan(engine, N, H, W, C, K, G, R, S, filt, bias, act=act, stride=self.stride, padding=self.padding)
        self._own(engine, plan, filt, bias)

    def _grads(self, dy, dx):
        self.engine.gconv_wgrad(self.plan, self._x, dy, self.dw)
        if dx is not None:
            self.engine.gconv_dgrad(self.plan, dy, dx)


class BatchNormLayer:
    """Batch normalization trained on the device (pcnn_batchnorm_nhwc_bf16_fwd / _bwd), as torch's BatchNorm2d with affine
    parameters, with an optional residual add and ReLU after it.  It owns fp32 gamma (default ones) and beta (default zeros), their
    gradients dgamma and dbeta, the running mean and variance (zeros and ones, updated with `momentum` by every training forward)
    and the saved mean and rstd of the last training forward, all in DeviceArrays.

    x, r, y, dy, dy2, dx and dr are dense bf16 [N][H][W][C]: what a ConvLayer writes as y and reads as dy.  act ACT_RELU (3) is
    a ReLU after the add, ACT_NONE (0) none; ACT_SILU (4), ACT_HARDSWISH (5) and ACT_RELU6 (6) are the activations of EfficientNet,
    MobileNetV3 and MobileNetV2, whose backward works from the pre-activation recomputed from x and r rather than from y, so at those
    codes the layer keeps r as well as x.  A ResNet basic block, x0 being a previous BatchNormLayer's output:

        conv_a.forward(x0, ya); bn_a.forward(ya, za); conv_b.forward(za, yb); bn_b.forward(yb, out, r=x0)
        bn_b.backward(out, dout, dyb, dr=dres); conv_b.backward(yb, dyb, dza); bn_a.backward(za, dza, dya)
        conv_a.backward(ya, dya, dx0)

    with bn_a at ACT_RELU, bn_b at ACT_RELU, conv_a and conv_b without bias; the BatchNormLayer that wrote x0 completes the join
    with backward(..., dx0, dy2=dres)."""

    def __init__(self, engine, N, H, W, C, act=0, eps=1e-5, momentum=0.1, gamma=None, beta=None):
        self.engine = engine
        self.shape = (N, H, W, C)
        self.pixels = int(N) * int(H) * int(W)
        self.act, self.eps, self.momentum = int(act), float(eps), float(momentum)
        self.info = batchnorm_nhwc_info(self.pixels, C, True)
        g = np.ones(C, np.float32) if gamma is None else np.ascontiguousarray(gamma, np.float32).reshape(C)
        b = np.zeros(C, np.float32) if beta is None else np.ascontiguousarray(beta, np.float32).reshape(C)
        self.gamma, self.beta = DeviceArray.from_host(engine, g), DeviceArray.from_host(engine, b)
        self.dgamma, self.dbeta = engine.array(C), engine.array(C)
        self.running_mean = DeviceArray.from_host(engine, np.zeros(C, np.float32))
        self.running_var = DeviceArray.from_host(engine, np.ones(C, np.float32))
        self.save_mean, self.save_rstd = engine.array(C), engine.array(C)
        self._x = self._r = None

    def forward(self, x, y, r=None, training=True):
        """y = act(bn(x) + r).  training: batch statistics, saved for backward, and the running statistics updated; otherwise the
        running statistics.  The layer keeps x (and r at ACT_SILU, ACT_HARDSWISH and ACT_RELU6): backward reads them, so they must
        stay unchanged until then."""
        N, H, W, C = self.shape
        self.engine.batchnorm_fwd(x, y, self.pixels, C, self.gamma, self.beta, self.running_mean, self.running_var, self.save_mean,
                                  self.save_rstd, r=r, act=self.act, training=training, eps=self.eps, momentum=self.momentum)
        if training:
            self._x = x
            if self.act in PREACT_CODES:
                self._r = r

    def backward(self, y, dy, dx, dr=None, dy2=None):
        """Gradients of the most recent training forward, whose output y was: dgamma, dbeta and dx (dx may be dy).  dy2 is a second
        gradient added to dy before the activation (the other branch of a residual join); dr receives the gradient of the
        forward's r.  At ACT_SILU, ACT_HARDSWISH and ACT_RELU6 y is not read: the gradient is taken at the recomputed
        pre-activation (Engine.batchnorm_bwd_preact)."""
        N, H, W, C = self.shape
        if self.act in PREACT_CODES:
            self.engine.batchnorm_bwd_preact(self._x, dy, self.gamma, self.beta, self.save_mean, self.save_rstd, dx, self.dgamma, self.dbeta,
                                             self.pixels, C, self.act, r=self._r, dy2=dy2, dr=dr)
            return
        self.engine.batchnorm_bwd(self._x, y, dy, self.gamma, self.save_mean, self.save_rstd, dx, self.dgamma, self.dbeta, self.pixels, C,
                                  act=self.act, dy2=dy2, dr=dr)

    def sgd(self, lr):
        """gamma += (-lr) * dgamma and beta += (-lr) * dbeta in fp32, on the engine's stream"""
        C = self.shape[3]
        self.engine.apply_grad_scaled(self.gamma, self.dgamma, C, -lr)
        self.engine.apply_grad_scaled(self.beta, self.dbeta, C, -lr)

    def optim_tensors(self):
        """(param, grad, plan, plan part, is norm or bias) of gamma and beta, as ConvLayer.optim_tensors"""
        return [(self.gamma, self.dgamma, None, 0, True), (self.beta, self.dbeta, None, 0, True)]

    def params(self):
        """host copies of gamma, beta, the running mean and the running variance"""
        return self.gamma.to_host(), self.beta.to_host(), self.running_mean.to_host(), self.running_var.to_host()

    def close(self):
        for a in (self.gamma, self.beta, self.dgamma, self.dbeta, self.running_mean, self.running_var, self.save_mean, self.save_rstd):
            a.free()


class GroupNormLayer:
    """Group normalization trained on the device (pcnn_groupnorm_nhwc_bf16_fwd / _bwd / _bwd_preact), as torch's GroupNorm with
    affine parameters, with BatchNormLayer's residual add and activations after it.  The statistics are those of each image's
    groups of C / groups channels, so one image's output never depends on another's, and there are no running statistics:
    forward takes no training flag.  It owns fp32 gamma (default ones) and beta (default zeros), their gradients dgamma and dbeta,
    the saved mean and rstd [N][groups] of the last forward and the group sums dstat [2][N][groups] of the last backward, all in
    DeviceArrays.

    x, r, y, dy, dy2, dx and dr are dense bf16 [N][H][W][C], as for a BatchNormLayer, which this layer replaces where a batch
    holds few images (segmentation, detection heads).  At ACT_SILU, ACT_HARDSWISH and ACT_RELU6 the backward works from the
    pre-activation recomputed from x and r, so at those codes the layer keeps r as well as x."""

    def __init__(self, engine, N, H, W, C, groups, act=0, eps=1e-5, gamma=None, beta=None):
        self.engine = engine
        self.shape = (N, H, W, C)
        self.groups, self.HW = int(groups), int(H) * int(W)
        self.act, self.eps = int(act), float(eps)
        self.info = groupnorm_nhwc_info(N, self.HW, C, self.groups)
        g = np.ones(C, np.float32) if gamma is None else np.ascontiguousarray(gamma, np.float32).reshape(C)
        b = np.zeros(C, np.float32) if beta is None else np.ascontiguousarray(beta, np.float32).reshape(C)
        self.gamma, self.beta = DeviceArray.from_host(engine, g), DeviceArray.from_host(engine, b)
        self.dgamma, self.dbeta = engine.array(C), engine.array(C)
        self.save_mean, self.save_rstd = engine.array(N * self.groups), engine.array(N * self.groups)
        self.dstat = engine.array(2 * N * self.groups)
        self._x = self._r = None

    def forward(self, x, y, r=None):
        """y = act(gn(x) + r), the statistics saved for backward.  The layer keeps x (and r at ACT_SILU, ACT_HARDSWISH and
        ACT_RELU6): backward reads them, so they must stay unchanged until then."""
        N, H, W, C = self.shape
        self.engine.groupnorm_fwd(x, y, N, self.HW, C, self.groups, self.gamma, self.beta, self.save_mean, self.save_rstd, r=r,
                                  act=self.act, eps=self.eps)
        self._x = x
        self._r = r if self.act in PREACT_CODES else None

    def backward(self, y, dy, dx, dr=None, dy2=None):
        """Gradients of the most recent forward, whose output y was: dgamma, dbeta, dstat and dx (dx may be dy).  dy2 is a second
        gradient added to dy before the activation; dr receives the gradient of the forward's r.  At ACT_SILU, ACT_HARDSWISH and
        ACT_RELU6 y is not read (Engine.groupnorm_bwd_preact)."""
        N, H, W, C = self.shape
        if self.act in PREACT_CODES:
            self.engine.groupnorm_bwd_preact(self._x, dy, self.gamma, self.beta, self.save_mean, self.save_rstd, dx, self.dgamma,
                                             self.dbeta, self.dstat, N, self.HW, C, self.groups, self.act, r=self._r, dy2=dy2, dr=dr)
            return
        self.engine.groupnorm_bwd(self._x, y, dy, self.gamma, self.save_mean, self.save_rstd, dx, self.dgamma, self.dbeta, self.dstat, N,
                                  self.HW, C, self.groups, act=self.act, dy2=dy2, dr=dr)

    def sgd(self, lr):
        """gamma += (-lr) * dgamma and beta += (-lr) * dbeta in fp32, on the engine's stream"""
        C = self.shape[3]
        self.engine.apply_grad_scaled(self.gamma, self.dgamma, C, -lr)
        self.engine.apply_grad_scaled(self.beta, self.dbeta, C, -lr)

    def optim_tensors(self):
        """(param, grad, plan, plan part, is norm or bias) of gamma and beta, as BatchNormLayer.optim_tensors"""
        return [(self.gamma, self.dgamma, None, 0, True), (self.beta, self.dbeta, None, 0, True)]

    def params(self):
        """host copies of gamma and beta"""
        return self.gamma.to_host(), self.beta.to_host()

    def close(self):
        for a in (self.gamma, self.beta, self.dgamma, self.dbeta, self.save_mean, self.save_rstd, self.dstat):
            a.free()


class LinearLayer(_PlanLayer):
    """A fully connected layer trained on the device, with ConvLayer's interface: fp32 masters w [O][P][Q][C] and bias [O], their
    gradients dw and db, and a LinearPlan holding w in bf16.

    x is [N][image_rows][row_pitch] bf16 with P x Q pixels of C channels per image, which is what MaxPoolLayer writes as y (pass
    its row_pitch and image_rows) or, with P = Q = 1 and C = the previous O, what a LinearLayer writes (row_pitch = that O, a
    multiple of 8).  y and dy are dense [N][O]; dx is written in x's layout.  act ACT_SIGMOID (1) is a sigmoid after the bias,
    ACT_RELU (3) a ReLU, ACT_NONE (0) none.  A LeNet-style
    classifier runs every pass on the engine's stream:

        conv1.forward(x, y1);  pool1.forward(y1, x2);  conv2.forward(x2, y2);  pool2.forward(y2, x3)
        fc1.forward(x3, y3);  fc2.forward(y3, z)
        engine.softmax_ce_bf16(z, labels, N, 10, 1 / N, dz, loss, pred)
        fc2.backward(z, dz, dy3);  fc1.backward(y3, dy3, dx3);  pool2.backward(dx3, dy2)
        conv2.backward(y2, dy2, dx2);  pool1.backward(dx2, dy1);  conv1.backward(y1, dy1, None)
        for layer in (conv1, conv2, fc1, fc2): layer.sgd(lr)

    dx uses the plan's bf16 weights, so call backward before sgd."""

    def __init__(self, engine, N, P, Q, C, O, w, bias=None, act=0, row_pitch=None, image_rows=0):
        self.shape = (N, P, Q, C, O)
        self.act = int(act)
        self.row_pitch = int(row_pitch or (Q * C + 7) // 8 * 8)
        self.image_rows = int(image_rows)
        self.info = linear_info(N, P, Q, C, O, self.row_pitch, self.image_rows)
        w = np.ascontiguousarray(w, np.float32).reshape(O, P, Q, C)
        bias = None if bias is None else np.ascontiguousarray(bias, np.float32).reshape(O)
        plan = LinearPlan(engine, N, P, Q, C, O, w, bias, act=act, row_pitch=self.row_pitch, image_rows=self.image_rows)
        self._own(engine, plan, w, bias)

    @property
    def w(self):
        """the fp32 master weights [O][P][Q][C]"""
        return self.filt

    def _grads(self, dy, dx):
        self.engine.linear_wgrad(self.plan, self._x, dy, self.dw)
        if dx is not None:
            self.engine.linear_dgrad(self.plan, dy, dx)


class SelfAttentionLayer:
    """Multi-head self-attention over the H x W pixels of each image, trained on the device: a fused qkv LinearLayer (C -> 3 heads
    head_dim, so heads * head_dim <= 85), the attention core (pcnn_attention_bf16_fwd / _bwd) and an output LinearLayer (heads
    head_dim -> C).  w_qkv is fp32 [3 heads head_dim][C] with the rows of q, then k, then v, head j at rows j head_dim of each; w_out
    is [C][heads head_dim].  scale None = 1 / sqrt(head_dim).

    x, y, dy and dx are dense bf16 [N][H][W][C] (C a multiple of 8).  The residual and the normalization of a non-local block stay in
    the network, joined through dy2 as every residual here is:

        attn.forward(x, wz);  bn.forward(wz, z, r=x)
        bn.backward(z, dz, dwz, dr=dres);  attn.backward(dwz, dx);  <the layer that wrote x>.backward(..., dx, dy2=dres)

    The layer keeps x and its own activations (qkv, o, lse) for backward.  optim_tensors() lists both projections' tensors, so SGD
    and AdamW take the layer as they take a LinearLayer."""

    def __init__(self, engine, N, H, W, C, heads, head_dim, w_qkv, b_qkv, w_out, b_out=None, scale=None):
        self.engine = engine
        self.shape = (N, H, W, C)
        self.heads, self.d = int(heads), int(head_dim)
        self.T = int(H) * int(W)
        self.scale = 1.0 / math.sqrt(self.d) if scale is None else float(scale)
        hd = self.heads * self.d
        rows = int(N) * self.T
        self.info = attention_info(N, self.T, self.heads, self.d, 3 * hd, 3 * hd, self.scale)
        self.qkv = LinearLayer(engine, rows, 1, 1, C, 3 * hd, w_qkv, b_qkv)
        self.out = LinearLayer(engine, rows, 1, 1, hd, C, w_out, b_out)
        self.qkv_y, self.dqkv = engine.array(rows * 3 * hd, np.uint16), engine.array(rows * 3 * hd, np.uint16)
        self.o, self.do = engine.array(rows * hd, np.uint16), engine.array(rows * hd, np.uint16)
        self.lse = engine.array(int(N) * self.heads * self.T)

    def _qkv(self, base):
        hd2 = self.heads * self.d * 2
        return base.ptr, base.ptr + hd2, base.ptr + 2 * hd2

    def forward(self, x, y):
        """y = out(attention(qkv(x))) + b_out"""
        N, H, W, C = self.shape
        self.qkv.forward(x, self.qkv_y)
        self.engine.attention_fwd(*self._qkv(self.qkv_y), self.o, self.lse, N, self.T, self.heads, self.d, ld=3 * self.heads * self.d,
                                  scale=self.scale)
        self.out.forward(self.o, y)

    def backward(self, dy, dx):
        """Gradients of the most recent forward: both projections' dw and db and, when dx is given, dx.  dy is left unchanged."""
        N, H, W, C = self.shape
        ld = 3 * self.heads * self.d
        self.out.backward(None, dy, self.do)
        self.engine.attention_bwd(*self._qkv(self.qkv_y), self.o, self.do, self.lse, *self._qkv(self.dqkv), N, self.T, self.heads, self.d,
                                  ld=ld, ld_g=ld, scale=self.scale)
        self.qkv.backward(None, self.dqkv, dx)

    def sgd(self, lr):
        self.qkv.sgd(lr)
        self.out.sgd(lr)

    def optim_tensors(self):
        """the qkv projection's tensors, then the output projection's, as LinearLayer.optim_tensors"""
        return self.qkv.optim_tensors() + self.out.optim_tensors()

    def params(self):
        """host copies (w_qkv, b_qkv, w_out, b_out) of the fp32 masters; b_out None without one"""
        return (*self.qkv.params(), *self.out.params())

    def close(self):
        self.qkv.close()
        self.out.close()
        for a in (self.qkv_y, self.dqkv, self.o, self.do, self.lse):
            a.free()


class MaxPoolLayer:
    """Max pooling between two ConvLayers (pcnn_maxpool_nhwc_bf16_fwd / _bwd), as max_pool2d(kernel (R, S), stride, padding): S
    defaults to R and stride to R, as torch does.  It owns the uint8 argmax [N][P][Q][C] the backward reads.

    x is what a ConvLayer's forward writes as y (dense [N][H][W][C]); y is written in the layout the next layer reads as x
    (row_pitch None = Q*C rounded up to 8, image_rows 0 = P: pass that layer's row_pitch and image_rows); dx is what the
    previous layer's backward reads as dy.  A stack runs with no copies:

        conv1.forward(x, y1);  pool.forward(y1, x2);  conv2.forward(x2, y2)
        conv2.backward(y2, dy2, dx2);  pool.backward(dx2, dy1);  conv1.backward(y1, dy1, None)

    with x2 and dx2 in conv2's x layout and y1 and dy1 dense [N][H][W][C]."""

    def __init__(self, engine, N, H, W, C, R, S=None, stride=None, padding=(0, 0), row_pitch=None, image_rows=0):
        self.engine = engine
        S = R if S is None else S
        stride = R if stride is None else stride
        self.shape = (N, H, W, C, R, S)
        self.stride = int(stride)
        self.padding = tuple(int(v) for v in padding)
        info = maxpool_nhwc_info(N, H, W, C, R, S, self.stride, self.padding, row_pitch or 0, image_rows)
        self.row_pitch, self.image_rows = info["row_pitch"], int(image_rows)
        self.out_shape = (N, info["P"], info["Q"], C)
        self.argmax = engine.array(self.out_shape, np.uint8)

    def forward(self, x, y):
        """y = max over each window of x, and the argmax the backward reads"""
        self.engine.maxpool_nhwc_fwd(x, y, self.argmax, *self.shape, self.stride, self.padding, self.row_pitch, self.image_rows)

    def backward(self, dy, dx):
        """dx (dense, every element written) from dy (in y's layout) through the argmax of the most recent forward"""
        self.engine.maxpool_nhwc_bwd(dy, self.argmax, dx, *self.shape, self.stride, self.padding, self.row_pitch, self.image_rows)

    def close(self):
        self.argmax.free()


class AvgPoolLayer:
    """Average pooling between two layers (pcnn_avgpool_nhwc_bf16_fwd / _bwd), as avg_pool2d(kernel (R, S), stride, padding,
    count_include_pad=count_include_pad): S defaults to R and stride to R, as torch does.  Layouts as MaxPoolLayer: x dense
    [N][H][W][C], y in the layout the next layer reads as x (row_pitch None = Q*C rounded up to 8, image_rows 0 = P), dx dense.
    It keeps no state: the backward reads dy alone."""

    def __init__(self, engine, N, H, W, C, R, S=None, stride=None, padding=(0, 0), count_include_pad=True, row_pitch=None, image_rows=0):
        self.engine = engine
        S = R if S is None else S
        stride = R if stride is None else stride
        self.shape = (N, H, W, C, R, S)
        self.stride = int(stride)
        self.padding = tuple(int(v) for v in padding)
        self.count_include_pad = bool(count_include_pad)
        info = avgpool_nhwc_info(N, H, W, C, R, S, self.stride, self.padding, row_pitch or 0, image_rows)
        self.row_pitch, self.image_rows = info["row_pitch"], int(image_rows)
        self.out_shape = (N, info["P"], info["Q"], C)

    def forward(self, x, y):
        """y = the mean of each window of x"""
        self.engine.avgpool_nhwc_fwd(x, y, *self.shape, self.stride, self.padding, self.count_include_pad, self.row_pitch, self.image_rows)

    def backward(self, dy, dx):
        """dx (dense, every element written) from dy (in y's layout)"""
        self.engine.avgpool_nhwc_bwd(dy, dx, *self.shape, self.stride, self.padding, self.count_include_pad, self.row_pitch, self.image_rows)

    def close(self):
        pass


class GlobalAvgPoolLayer:
    """Global average pooling (pcnn_global_avgpool_nhwc_bf16_fwd / _bwd), as adaptive_avg_pool2d(x, 1): x and dx dense bf16
    [N][H][W][C], y and dy [N][row_pitch] (row_pitch None = C rounded up to 8), the x layout of LinearLayer(engine, N, 1, 1, C, O).
    It keeps no state; info is its partition (global_avgpool_nhwc_info)."""

    def __init__(self, engine, N, H, W, C, row_pitch=None):
        self.engine = engine
        self.shape = (N, H, W, C)
        self.info = global_avgpool_nhwc_info(N, H, W, C, row_pitch or 0)
        self.row_pitch = self.info["row_pitch"]
        self.out_shape = (N, C)

    def forward(self, x, y):
        """y[n][c] = the mean of x[n][:, :, c].  The head of a ResNet, z being a BatchNormLayer's output:

            bn.forward(yc, z);  gap.forward(z, h);  fc.forward(h, logits)
            engine.softmax_ce_bf16(logits, labels, N, O, 1 / N, dlogits)

        with fc = LinearLayer(engine, N, 1, 1, C, O, w, b, row_pitch=gap.row_pitch) and h [N][gap.row_pitch]."""
        self.engine.global_avgpool_nhwc_fwd(x, y, *self.shape, self.row_pitch)

    def backward(self, dy, dx):
        """dx = dy / (H*W) at every pixel: the chain of forward runs back as

            fc.backward(logits, dlogits, dh);  gap.backward(dh, dz);  bn.backward(z, dz, dyc)

        with dh in h's layout (its pad never read) and dz dense [N][H][W][C]."""
        self.engine.global_avgpool_nhwc_bwd(dy, dx, *self.shape, self.row_pitch)

    def close(self):
        pass


class DropoutLayer:
    """Dropout (per_sample False: each element dropped with probability p) or stochastic depth (per_sample True: each row, an
    image, dropped whole) on the device (pcnn_dropout_bf16): y = x * m (+ r), m = 0 or 1 / (1 - p).  x, r, y, dy and dx are N bf16
    rows of row_elems elements, row_pitch apart (None = dense): a dense NHWC activation (row_elems = H*W*C), a GlobalAvgPoolLayer's
    output (row_elems = C, row_pitch = gap.row_pitch) or a dense LinearLayer output [N][O].  It has no parameters, so no
    optim_tensors.

    The mask of a training forward is the Philox draw of (seed, call) at each index, call being incremented by every training
    forward; `call` is a plain attribute, so a checkpoint can save and restore it and replay the same masks.  backward applies the
    mask of the most recent training forward.  Dropout in place before a classifier:

        gap.forward(z, h);  drop.forward(h, h);  fc.forward(h, logits)
        fc.backward(logits, dlogits, dh);  drop.backward(dh, dh);  gap.backward(dh, dz)

    Stochastic depth on a residual block: the branch's last batch norm runs without r, and the layer adds the skip path:

        bn.forward(yb, b)                   # the branch's last BN, without r
        drop.forward(b, out, r=x_in)        # out = x_in + drop_path(b)
        drop.backward(dout, db)             # dout still feeds the skip path as dy2

    dx may be dy (in place), but not when dy is still needed, as here, where dout is also the gradient of x_in."""

    def __init__(self, engine, N, row_elems, p, seed, per_sample=False, row_pitch=None):
        self.info = dropout_info(N, row_elems, row_pitch or 0, p, per_sample)
        self.engine = engine
        self.shape = (int(N), int(row_elems))
        self.row_pitch = int(row_pitch or 0)
        self.p, self.seed, self.per_sample = float(p), int(seed), bool(per_sample)
        self.call = 0

    def forward(self, x, y, r=None, training=True):
        """training: call += 1, then y = x * m (+ r) with this call's mask.  Eval: y = x (+ r), nothing launched when y is x and
        there is no r.  y may be x or r."""
        if training:
            self.call += 1
            self.engine.dropout(x, y, *self.shape, self.p, self.seed, self.call, self.per_sample, r=r, row_pitch=self.row_pitch)
        elif r is not None or _p(y) != _p(x):
            self.engine.dropout(x, y, *self.shape, 0.0, self.seed, 0, False, r=r, row_pitch=self.row_pitch)

    def backward(self, dy, dx):
        """dx = dy * m, the mask of the most recent training forward (the gradient of r is dy itself).  dx may be dy."""
        if self.call == 0:
            raise PcnnError("DropoutLayer.backward", -1, "no training forward has drawn a mask (call = 0)")
        self.engine.dropout(dy, dx, *self.shape, self.p, self.seed, self.call, self.per_sample, row_pitch=self.row_pitch)

    def close(self):
        pass


class ImageBatcher:
    """The input path of a device-trained network (pcnn_augment_u8_bf16): a uint8 dataset [n][H][W] or [n][H][W][C] (a device
    tensor, a DeviceArray, or a host array uploaded once) and its uint8 labels [n] (or None) become batches of N images in the x
    layout a plan reads, in one launch per batch.  Training batches take the epoch in a fresh order (shuffle), each image cropped
    from the image zero-padded by pad (RandomCrop) and mirrored with probability 1/2 (flip), then normalised per channel by mean /
    std (None = 0 / 1, a scalar for every channel).  x has C_out channels (None = C) at row_pitch / image_rows (0 = dense), so a
    network's first layer reads it as it is: for the example networks' MNIST layer, C_out 1, row_pitch 32, image_rows 28.

    The batcher owns x and the label buffer; batch(step) overwrites them in stream order and returns (x pointer, labels), the
    arguments of the networks' forward(x, labels).  Everything random is a function of (seed, epoch, dataset index), so a
    checkpoint that saves `epoch`, a plain attribute the caller sets, replays the same batches.  The last partial batch of an
    epoch is dropped: steps_per_epoch = n // N.

        for ep in range(epochs):
            batcher.epoch = ep
            for s in range(batcher.steps_per_epoch):
                net.forward(*batcher.batch(s)); net.backward(); net.sgd(lr)
        net.forward(*test_batcher.batch(0, training=False), training=False)

    batch(step, training=False) is the eval path: identity order, no crop and no flip.

    mixup_alpha / cutmix_alpha > 0 mix every training batch (pcnn_augment_mix_u8_bf16) with the MixUp or CutMix that
    mix_draws(seed, epoch, step, ...) picks, and batch(step) then returns (x pointer, MixedLabels), the batcher owning labels_b;
    softmax_ce_soft_bf16 takes those targets.  Both 0 (the default) is the plain batcher, bit for bit.

    crop_size (an int or (h, w)) resizes (pcnn_augment_resized_u8_bf16): training batches take torchvision's
    RandomResizedCrop(crop_size, scale, ratio, antialias=True) and the flip, eval batches Resize(resize_size) +
    CenterCrop(crop_size), resize_size defaulting to the crop's shorter side; x then holds crop_size pixels per image.  It excludes
    pad > 0 and mixing.  crop_size None (the default) is the plain batcher, bit for bit.

    trivial_augment "nearest" or "bilinear" and random_erase > 0 (a probability, with erase_scale and erase_ratio) add
    torchvision's TrivialAugmentWide after the crop and flip and RandomErasing(value=0) after Normalize to training batches
    (pcnn_augment_trivial_u8_bf16), the batcher owning the uint8 workspace between its two launches.  TrivialAugmentWide needs
    C 1 or 3; neither excludes crop_size, both exclude mixing.  Eval batches are unchanged.  trivial_augment None with
    random_erase 0 (the defaults) is the batcher without them, bit for bit."""

    def __init__(self, engine, images, labels, N, pad=0, flip=False, shuffle=True, seed=0, mean=None, std=None, C_out=None,
                 row_pitch=0, image_rows=0, mixup_alpha=0.0, cutmix_alpha=0.0, crop_size=None, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3),
                 resize_size=None, trivial_augment=None, random_erase=0.0, erase_scale=(0.02, 0.33), erase_ratio=(0.3, 3.3), masks=None,
                 mask_fill=255):
        if masks is not None:
            if crop_size is not None or trivial_augment is not None or random_erase != 0 or mixup_alpha != 0 or cutmix_alpha != 0:
                raise PcnnError("ImageBatcher", -1, "masks with crop_size, trivial_augment, random_erase or mixing: masks are carried "
                                "through the plain crop, pad and flip only")
            mshape = tuple(int(d) for d in masks.shape)
            if mshape != tuple(int(d) for d in images.shape[:3]) or "uint8" not in str(masks.dtype):
                raise PcnnError("ImageBatcher", -1, f"masks must be uint8 [n][H][W] = {tuple(images.shape[:3])}, got {masks.dtype} {mshape}")
            if not (isinstance(mask_fill, (int, np.integer)) and 0 <= mask_fill <= 255):
                raise PcnnError("ImageBatcher", -1, f"mask_fill = {mask_fill}: an integer 0 .. 255 is required")
        modes = {None: TRIVIAL_NONE, "nearest": TRIVIAL_NEAREST, "bilinear": TRIVIAL_BILINEAR}
        if not isinstance(trivial_augment, (str, type(None))) or trivial_augment not in modes:
            raise PcnnError("ImageBatcher", -1, f"trivial_augment = {trivial_augment!r}: None, 'nearest' or 'bilinear' is required")
        if not (isinstance(random_erase, (int, float, np.integer, np.floating)) and math.isfinite(random_erase) and 0 <= random_erase <= 1):
            raise PcnnError("ImageBatcher", -1, f"random_erase = {random_erase}: a probability 0 <= p <= 1 is required")
        self.trivial, self.random_erase = modes[trivial_augment], float(random_erase)
        self.erase_scale, self.erase_ratio = (float(erase_scale[0]), float(erase_scale[1])), (float(erase_ratio[0]), float(erase_ratio[1]))
        self.augmenting = self.trivial != TRIVIAL_NONE or self.random_erase > 0
        if self.augmenting and (mixup_alpha > 0 or cutmix_alpha > 0):
            raise PcnnError("ImageBatcher", -1, "trivial_augment or random_erase with mixup_alpha or cutmix_alpha > 0: these batches are "
                            "not mixed")
        for name, a in (("mixup_alpha", mixup_alpha), ("cutmix_alpha", cutmix_alpha)):
            if not (isinstance(a, (int, float, np.integer, np.floating)) and math.isfinite(a) and a >= 0):
                raise PcnnError("ImageBatcher", -1, f"{name} = {a}: a finite alpha >= 0 is required")
        self.mixup_alpha, self.cutmix_alpha = float(mixup_alpha), float(cutmix_alpha)
        self.mixing = self.mixup_alpha > 0 or self.cutmix_alpha > 0
        if self.mixing and labels is None:
            raise PcnnError("ImageBatcher", -1, "mixup_alpha or cutmix_alpha > 0 needs labels to mix")
        self.crop = None if crop_size is None else tuple(int(v) for v in np.broadcast_to(np.asarray(crop_size).reshape(-1), (2,)))
        if self.crop is not None and int(pad) > 0:
            raise PcnnError("ImageBatcher", -1, f"crop_size = {crop_size} with pad = {pad}: a resized batch takes no padding")
        if self.crop is not None and self.mixing:
            raise PcnnError("ImageBatcher", -1, f"crop_size = {crop_size} with mixup_alpha or cutmix_alpha > 0: resized batches are not mixed")
        if self.crop is None and resize_size is not None:
            raise PcnnError("ImageBatcher", -1, f"resize_size = {resize_size} without crop_size: only a resized batcher resizes")
        self.scale, self.ratio = (float(scale[0]), float(scale[1])), (float(ratio[0]), float(ratio[1]))
        self.resize_size = None if self.crop is None else int(min(self.crop) if resize_size is None else resize_size)
        shape = tuple(int(d) for d in images.shape)
        if len(shape) not in (3, 4):
            raise PcnnError("ImageBatcher", -1, f"images must be [n][H][W] or [n][H][W][C], got shape {shape}")
        if "uint8" not in str(images.dtype):
            raise PcnnError("ImageBatcher", -1, f"images must be uint8, got {images.dtype}")
        self.n, self.H, self.W = shape[:3]
        self.C = shape[3] if len(shape) == 4 else 1
        self.N, self.pad, self.flip, self.shuffle, self.seed = int(N), int(pad), bool(flip), bool(shuffle), int(seed)
        self.mean, self.std = channel_stats(mean, self.C, "mean"), channel_stats(std, self.C, "std")
        self.C_out = self.C if C_out is None else int(C_out)
        if self.crop is None:
            self.info, self.lut = augment_info(self.n, self.H, self.W, self.C, 0, self.N, int(self.shuffle), self.pad, int(self.flip),
                                               self.C_out, row_pitch, image_rows, self.mean, self.std)
        else:
            self.info, self.lut = augment_resized_info(self.n, self.H, self.W, self.C, 0, self.N, *self.crop, RESIZE_TRAIN, self.scale,
                                                       self.ratio, 0, int(self.shuffle), int(self.flip), self.C_out, row_pitch,
                                                       image_rows, self.mean, self.std)
            augment_resized_info(self.n, self.H, self.W, self.C, 0, self.N, *self.crop, RESIZE_EVAL, resize_size=self.resize_size,
                                 C_out=self.C_out, row_pitch=row_pitch, image_rows=image_rows, mean=self.mean, std=self.std)
        self.ws_info = None
        if self.augmenting:
            self.ws_info = augment_trivial_info(self.n, self.H, self.W, self.C, 0, self.N, self.trivial, self.random_erase,
                                                self.erase_scale, self.erase_ratio, self.crop, self.scale, self.ratio, int(self.shuffle),
                                                self.pad, int(self.flip), self.C_out, row_pitch, image_rows, self.mean, self.std)[0]
        if labels is not None and int(labels.shape[0]) != self.n:
            raise PcnnError("ImageBatcher", -1, f"{labels.shape[0]} labels for {self.n} images")
        self.engine = engine
        self.images = engine.to_device(images) if isinstance(images, np.ndarray) else images
        self.labels = engine.to_device(np.asarray(labels, np.uint8)) if isinstance(labels, np.ndarray) else labels
        self.x = engine.array((self.N, self.info["image_rows"], self.info["row_pitch"]), np.uint16)    # zeroed: the pad stays 0
        self.labels_out = engine.array((self.N,), np.uint8) if labels is not None else None
        self.labels_b = engine.array((self.N,), np.uint8) if self.mixing else None
        self.workspace = engine.array((self.ws_info["ws_bytes"],), np.uint8) if self.augmenting else None
        self.mask_fill = int(mask_fill)
        self.masks = None if masks is None else engine.to_device(np.ascontiguousarray(masks, np.uint8)) if isinstance(masks, np.ndarray) else masks
        self.masks_out = None if masks is None else engine.array((self.N, self.H, self.W), np.uint8)
        self.steps_per_epoch = self.n // self.N
        self.epoch = 0

    def batch(self, step, training=True):
        """(x pointer, labels) of batch `step` of epoch self.epoch: positions step N .. step N + N - 1; a mixing batcher's training
        batches return (x pointer, MixedLabels), a batcher with masks (x pointer, labels, masks_out)"""
        if not 0 <= int(step) < self.steps_per_epoch:
            raise PcnnError("ImageBatcher.batch", -1, f"step = {step}: 0 <= step < steps_per_epoch = {self.steps_per_epoch} is required")
        aug = bool(training)
        args = (self.images, self.labels, self.n, self.H, self.W, self.C, int(step) * self.N, self.N, self.x, self.labels_out)
        kw = dict(shuffle=int(aug and self.shuffle), pad=self.pad if aug else 0, flip=int(aug and self.flip), seed=self.seed,
                  epoch=self.epoch, mean=self.mean, std=self.std, C_out=self.C_out, row_pitch=self.info["row_pitch"],
                  image_rows=self.info["image_rows"])
        if aug and self.augmenting:
            self.engine.augment_trivial(*args[:9], self.workspace, self.labels_out, trivial=self.trivial, erase_p=self.random_erase,
                                        erase_scale=self.erase_scale, erase_ratio=self.erase_ratio, crop_size=self.crop, scale=self.scale,
                                        ratio=self.ratio, **kw)
            return self.x.ptr, self.labels_out
        if self.crop is not None:
            del kw["pad"]
            self.engine.augment_resized(*args[:9], *self.crop, self.labels_out, mode=RESIZE_TRAIN if aug else RESIZE_EVAL,
                                        scale=self.scale, ratio=self.ratio, resize_size=self.resize_size, **kw)
            return self.x.ptr, self.labels_out
        if not (aug and self.mixing):
            self.engine.augment(*args, **kw)
            if self.masks is None:
                return self.x.ptr, self.labels_out
            self.engine.augment_mask(self.masks, self.n, self.H, self.W, int(step) * self.N, self.N, self.masks_out, shuffle=kw["shuffle"],
                                     pad=kw["pad"], flip=kw["flip"], seed=self.seed, epoch=self.epoch, mask_fill=self.mask_fill)
            return self.x.ptr, self.labels_out, self.masks_out
        kind, lam, box, lam_adjusted = mix_draws(self.seed, self.epoch, step, self.H, self.W, self.mixup_alpha, self.cutmix_alpha)
        weight = lam if kind == "mixup" else lam_adjusted
        self.engine.augment_mix(*args, labels_b_out=self.labels_b, mode=MIX_MIXUP if kind == "mixup" else MIX_CUTMIX, lam=weight,
                                box=box or (0, 0, 0, 0), **kw)
        return self.x.ptr, MixedLabels(self.labels_out, self.labels_b, weight, kind, box)

    def close(self):
        for a in (self.x, self.labels_out, self.labels_b, self.workspace, self.masks_out):
            if a is not None:
                a.free()


class SqueezeExcitationLayer:
    """Squeeze-and-excitation trained on the device, with BatchNormLayer's interface: y = act(x * s + r) with the gate
    s = sigmoid(fc2(relu(fc1(GAP(x))))) per image and channel (pcnn_se_scale_nhwc_* for the gating, GlobalAvgPoolLayer and two
    LinearLayers for the squeeze branch).  x, r, y, dy, dy2, dx and dr are dense bf16 [N][H][W][C]: what a BatchNormLayer writes
    and reads.  w1 [hidden][C], b1 [hidden], w2 [C][hidden], b2 [C] are the fp32 masters of fc1 (ReLU) and fc2 (sigmoid); the layer
    owns them with the branch's small bf16 buffers: h (pooled x), a (fc1's y), s (the gate), ds, da and dh.  act ACT_RELU (3) is a
    ReLU after the add, ACT_NONE (0) none.  In an SE-ResNet basic block the block's last batch norm runs without r and ReLU and the
    SE layer carries both:

        conv_a.forward(x0, ya); bn_a.forward(ya, za); conv_b.forward(za, yb); bn_b.forward(yb, zb); se.forward(zb, out, r=x0)
        se.backward(out, dout, dzb, dr=dres); bn_b.backward(zb, dzb, dyb); ...

    Limits: hidden % 8 == 0 (fc2 reads a as rows of hidden), C <= 256 and hidden <= 256 (LinearLayer's O)."""

    def __init__(self, engine, N, H, W, C, hidden, w1, b1, w2, b2, act=0):
        if hidden % 8 or not 1 <= hidden <= 256 or not 1 <= C <= 256:
            raise PcnnError("SqueezeExcitationLayer", -1,
                            f"C = {C}, hidden = {hidden}: 1 <= C <= 256 and 8 <= hidden <= 256 with hidden % 8 == 0 are required (the "
                            "linear layers' O limit and row-pitch rule)")
        if int(act) not in (0, ACT_RELU):
            raise PcnnError("SqueezeExcitationLayer", -1, f"act {act}: 0 (none) or 3 (ReLU) is required")
        self.engine = engine
        self.shape = (N, H, W, C)
        self.hidden, self.act = int(hidden), int(act)
        self.info = se_scale_nhwc_info(N, H, W, C)
        self.gap = GlobalAvgPoolLayer(engine, N, H, W, C)
        self.row_pitch = self.gap.row_pitch
        self.fc1 = LinearLayer(engine, N, 1, 1, C, hidden, np.asarray(w1, np.float32).reshape(hidden, 1, 1, C), b1, act=ACT_RELU,
                               row_pitch=self.row_pitch)
        self.fc2 = LinearLayer(engine, N, 1, 1, hidden, C, np.asarray(w2, np.float32).reshape(C, 1, 1, hidden), b2, act=ACT_SIGMOID)
        bf = lambda *shape: engine.array(shape, np.uint16)
        self.h, self.dh = bf(N, self.row_pitch), bf(N, self.row_pitch)
        self.a, self.da = bf(N, hidden), bf(N, hidden)
        self.s, self.ds = bf(N, C), bf(N, C)
        self._x = None

    def forward(self, x, y, r=None):
        """y = act(x * s + r), s the gate of this x.  The layer keeps x: backward reads it."""
        N, H, W, C = self.shape
        self.gap.forward(x, self.h)
        self.fc1.forward(self.h, self.a)
        self.fc2.forward(self.a, self.s)
        self.engine.se_scale_fwd(x, self.s, y, N, H, W, C, r=r, act=self.act)
        self._x = x

    def backward(self, y, dy, dx, dr=None, dy2=None):
        """Gradients of the most recent forward, whose output y was: fc1's and fc2's dw and db, and dx, the gradient through both the
        scale and the squeeze branch.  dy2 is a second gradient added to dy before the activation; dr receives the gradient of the
        forward's r.  Without dr, dy is CONSUMED: it is overwritten in place by that gradient, as LinearLayer does.  dx may be dy."""
        N, H, W, C = self.shape
        e = self.engine
        g = dy if dr is None else dr
        e.se_scale_bwd_gate(self._x, y, dy, g, self.ds, N, H, W, C, dy2=dy2, act=self.act)
        self.fc2.backward(self.s, self.ds, self.da)
        self.fc1.backward(self.a, self.da, self.dh)
        e.se_scale_bwd_input(g, self.s, dx, N, H, W, C, dpool=self.dh, dpool_row_pitch=self.row_pitch)

    def sgd(self, lr):
        """plain SGD on both linear layers' masters, their plans refreshed (LinearLayer.sgd)"""
        self.fc1.sgd(lr)
        self.fc2.sgd(lr)

    def optim_tensors(self):
        """(param, grad, plan, plan part, is norm or bias) of w1, b1, w2 and b2, as ConvLayer.optim_tensors"""
        return self.fc1.optim_tensors() + self.fc2.optim_tensors()

    def params(self):
        """host copies of the fp32 masters w1 [hidden][1][1][C], b1, w2 [C][1][1][hidden], b2"""
        return self.fc1.params() + self.fc2.params()

    def close(self):
        for layer in (self.fc1, self.fc2, self.gap):
            layer.close()
        for a in (self.h, self.dh, self.a, self.da, self.s, self.ds):
            a.free()


class FusedOptimizer:
    """One fused update of many fp32 parameter tensors per step (pcnn_optim_*; the rules and their order are in include/pcnn.h).
    tensors: (param, grad, n, weight_decay, plan, plan part) with plan None (part 0) or the ConvPlan / LinearPlan / DepthwiseConvPlan
    whose filters (part 1) or bias (part 2) param is the master of; the plan's operands are refreshed by the step.  kind OPTIM_SGD or
    OPTIM_ADAMW.  SGD and
    AdamW build the table from layers; this class takes it directly."""

    def __init__(self, engine, kind, tensors, momentum=0.0, dampening=0.0, nesterov=False, betas=(0.9, 0.999), eps=1e-8):
        self.engine, self.opt = engine, None
        self.sizes = [int(t[2]) for t in tensors]
        tab = (OptimTensor * len(tensors))()
        for e, (param, grad, n, wd, plan, part) in zip(tab, tensors):
            e.param, e.grad, e.n, e.weight_decay, e.plan, e.plan_part = _p(param), _p(grad), int(n), float(wd), _plan(plan), int(part)
        cfg = OptimConfig(int(kind), float(momentum), float(dampening), int(bool(nesterov)), float(betas[0]), float(betas[1]), float(eps))
        h = C_.c_void_p()
        check("pcnn_optim_create", lib().pcnn_optim_create(engine.ctx, C_.byref(cfg), tab, len(tensors), C_.byref(h)))
        self.opt = h

    def step(self, lr):
        """one update of every tensor with learning rate lr (rounded to fp32), enqueued on the engine's stream after the backward
        passes; a row-Toeplitz plan's filters take a second launch"""
        check("pcnn_optim_step", lib().pcnn_optim_step(self.engine.ctx, self.opt, float(lr)))

    def state(self):
        """host copies of each tensor's state: (momentum buffer, None) for SGD with momentum, (m, v) for AdamW, (None, None) for
        SGD without momentum"""
        out = []
        for i, n in enumerate(self.sizes):
            ptrs = (C_.c_void_p(), C_.c_void_p())
            check("pcnn_optim_state", lib().pcnn_optim_state(self.opt, i, C_.byref(ptrs[0]), C_.byref(ptrs[1])))
            pair = []
            for p in ptrs:
                if not p.value:
                    pair.append(None)
                    continue
                a = np.empty(n, np.float32)
                check("pcnn_d2h", lib().pcnn_d2h(self.engine.ctx, a.ctypes.data, p.value, a.nbytes))
                pair.append(a)
            out.append(tuple(pair))
        return out

    def info(self):
        """pcnn_optim_info: tensors, elements, tensors on the 16-byte vector path, chunks, grid of the update kernel, steps taken"""
        v = (C_.c_long * 6)()
        check("pcnn_optim_info", lib().pcnn_optim_info(self.opt, v))
        return dict(tensors=v[0], elements=v[1], vector_tensors=v[2], chunks=v[3], grid=v[4], steps=v[5])

    @property
    def steps(self):
        return self.info()["steps"]

    def close(self):
        if self.opt and self.engine.ctx:
            lib().pcnn_optim_destroy(self.engine.ctx, self.opt)
        self.opt = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _plan(plan):
    """the pcnn_conv_plan handle of a ConvPlan / LinearPlan (or of a raw c_void_p), None for none"""
    plan = getattr(plan, "plan", plan)
    return getattr(plan, "value", plan)


def _layer_tensors(layers, weight_decay, decay_norm_and_bias):
    return [(param, grad, param.nbytes // 4, 0.0 if norm_or_bias and not decay_norm_and_bias else weight_decay, plan, part)
            for layer in layers for param, grad, plan, part, norm_or_bias in layer.optim_tensors()]


class SGD(FusedOptimizer):
    """torch.optim.SGD over the trainable tensors of ConvLayers, DepthwiseConvLayers, GroupedConvLayers, LinearLayers, BatchNormLayers and
    SqueezeExcitationLayers, in one launch
    per step with the layers' plans refreshed: step(lr) replaces every layer.sgd(lr) of a training step (momentum 0 and weight decay 0 give the same
    bits).  decay_norm_and_bias=False gives batch normalization's gamma and beta and the biases weight decay 0; the default decays
    every tensor, as torch.optim does with one parameter group."""

    def __init__(self, engine, layers, momentum=0.0, dampening=0.0, nesterov=False, weight_decay=0.0, decay_norm_and_bias=True):
        super().__init__(engine, OPTIM_SGD, _layer_tensors(layers, weight_decay, decay_norm_and_bias), momentum=momentum,
                         dampening=dampening, nesterov=nesterov)


class AdamW(FusedOptimizer):
    """torch.optim.AdamW (decoupled weight decay; weight_decay 0 is Adam) over the trainable tensors of the layers, as SGD"""

    def __init__(self, engine, layers, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, decay_norm_and_bias=True):
        super().__init__(engine, OPTIM_ADAMW, _layer_tensors(layers, weight_decay, decay_norm_and_bias), betas=betas, eps=eps)


def f32_to_bf16_bits(a):
    """numpy float32 -> uint16 bf16 bit patterns (round to nearest even), the rounding the kernels use; NaN -> the quiet NaN
    0x7FC0 (rounding the payload could carry into the exponent and the sign: 0x7FFFFFFF would become -0)"""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    u = u + 0x7FFF + ((u >> 16) & 1)
    return np.where(nan, 0x7FC0, u >> 16).astype(np.uint16)


def bf16_bits_to_f32(b):
    return (np.ascontiguousarray(b, np.uint16).astype(np.uint32) << 16).view(np.float32)


C_ = C
__all__ = ["Engine", "DeviceArray", "ConvPlan", "WideConvPlan", "LinearPlan", "ConvLayer", "LinearLayer", "MaxPoolLayer", "AvgPoolLayer", "GlobalAvgPoolLayer", "BatchNormLayer", "GroupNormLayer", "SelfAttentionLayer", "FusedOptimizer", "SGD", "AdamW", "f32_to_bf16_bits", "bf16_bits_to_f32", "TRAIN_SET", "TEST_SET", "U8", "F32"]
