"""ctypes declarations for every symbol of include/pcnn.h (kept in the same order as the header)."""
import ctypes as C
import math
import os
import re

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.environ.get("PCNN_LIB_PATH") or os.path.join(HERE, "libpcnn.so")
HEADER = os.path.join(ROOT, "include", "pcnn.h")

NPARAM = 2343
OFF = dict(c1w=(0, 150), c1b=(150, 156), s1w=(156, 172), s1b=(172, 173), fw=(173, 2333), fb=(2333, 2343))
U8, F32 = 0, 1
MODE_AUTO, MODE_GRAPH, MODE_PERSISTENT = 0, 1, 2
TRAIN_SET, TEST_SET = 0, 1
ACT_NONE, ACT_SIGMOID, ACT_RELU = 0, 1, 3     # PCNN_ACT_*: the `act` of the device-trained layers (2 is not a code)
ACT_SILU, ACT_HARDSWISH, ACT_RELU6 = 4, 5, 6  # taken by the normalizations only (BatchNormLayer, GroupNormLayer and their Engine calls)
OPTIM_SGD, OPTIM_ADAMW = 0, 1                 # PCNN_OPTIM_*: the `kind` of pcnn_optim_config
LOSS_MSE, LOSS_L1 = 0, 1                      # PCNN_LOSS_*: the `mode` of pcnn_regression_loss_bf16


class PcnnError(RuntimeError):
    """A libpcnn.so entry point returned a non-zero status (message = pcnn_last_error_string())."""

    def __init__(self, fn, code, msg):
        super().__init__(f"{fn} failed with status {code}: {msg}")
        self.fn, self.code, self.msg = fn, code, msg


_vp, _i, _l, _f, _sz = C.c_void_p, C.c_int, C.c_long, C.c_float, C.c_size_t
_pvp = C.POINTER(C.c_void_p)
_ll = C.c_longlong


class OptimTensor(C.Structure):
    """pcnn_optim_tensor"""
    _fields_ = [("param", _vp), ("grad", _vp), ("n", _l), ("weight_decay", _f), ("plan", _vp), ("plan_part", _i)]


class OptimConfig(C.Structure):
    """pcnn_optim_config"""
    _fields_ = [("kind", _i), ("momentum", _f), ("dampening", _f), ("nesterov", _i), ("beta1", _f), ("beta2", _f), ("eps", _f)]

# name -> argtypes (every function returns int unless listed in _RESTYPE)
_SIG = {
    "pcnn_version": [],
    "pcnn_last_error_string": [],
    "pcnn_create": [_pvp, _i, _vp],
    "pcnn_destroy": [_vp],
    "pcnn_sync": [_vp],
    "pcnn_device_info": [_vp, C.POINTER(_i), C.POINTER(_i), C.POINTER(_i), C.POINTER(_sz)],
    "pcnn_malloc": [_vp, _pvp, _sz],
    "pcnn_free": [_vp, _vp],
    "pcnn_memset0": [_vp, _vp, _sz],
    "pcnn_h2d": [_vp, _vp, _vp, _sz],
    "pcnn_d2h": [_vp, _vp, _vp, _sz],
    "pcnn_d2d": [_vp, _vp, _vp, _sz],
    "pcnn_init_params_reference": [_vp],
    "pcnn_set_params": [_vp, _vp],
    "pcnn_get_params": [_vp, _vp],
    "pcnn_get_grads": [_vp, _vp],
    "pcnn_params_dev": [_vp, _pvp],
    "pcnn_set_learning_rate": [_vp, _f],
    "pcnn_save_params": [_vp, C.c_char_p],
    "pcnn_load_params": [_vp, C.c_char_p],
    "pcnn_apply_step_function": [_vp, _vp, _vp, _l],
    "pcnn_make_error": [_vp, _vp, _vp, C.c_uint, _i],
    "pcnn_make_error_batch": [_vp, _vp, _vp, _vp, _i],
    "pcnn_apply_grad": [_vp, _vp, _vp, _l],
    "pcnn_apply_grad_scaled": [_vp, _vp, _vp, _l, _f],
    "pcnn_vector_norm": [_vp, _vp, _i, _i, _vp],
    "pcnn_fp_c1": [_vp, _vp, _vp, _vp, _vp, _i],
    "pcnn_fp_s1": [_vp, _vp, _vp, _vp, _vp, _i],
    "pcnn_fp_preact_f": [_vp, _vp, _vp, _vp, _i],
    "pcnn_fp_bias_f": [_vp, _vp, _vp, _i],
    "pcnn_bp_weight_f": [_vp, _vp, _vp, _vp, _i],
    "pcnn_bp_bias_f": [_vp, _vp, _vp, _i],
    "pcnn_bp_output_s1": [_vp, _vp, _vp, _vp, _i],
    "pcnn_bp_preact_s1": [_vp, _vp, _vp, _vp, _i],
    "pcnn_bp_weight_s1": [_vp, _vp, _vp, _vp, _i],
    "pcnn_bp_bias_s1": [_vp, _vp, _vp, _i],
    "pcnn_bp_output_c1": [_vp, _vp, _vp, _vp, _i],
    "pcnn_bp_preact_c1": [_vp, _vp, _vp, _vp, _i],
    "pcnn_bp_weight_c1": [_vp, _vp, _vp, _vp, _i],
    "pcnn_bp_bias_c1": [_vp, _vp, _vp, _i],
    "pcnn_mnist_load_u8": [C.c_char_p, C.c_char_p, _pvp, _pvp, C.POINTER(C.c_uint)],
    "pcnn_mnist_free": [_vp],
    "pcnn_dataset_upload": [_vp, _i, _vp, _i, _vp, _l],
    "pcnn_dataset_bind": [_vp, _i, _vp, _i, _vp, _l],
    "pcnn_train_step": [_vp, _l, _i],
    "pcnn_train_steps": [_vp, _l, _i, _i],
    "pcnn_train_steps_prepare": [_vp, _i, _i],
    "pcnn_train_step_dev": [_vp, _vp, _i, _vp, _i],
    "pcnn_train_step_host": [_vp, _vp, _i, _vp, _i, C.POINTER(_f)],
    "pcnn_compute_grads": [_vp, _vp, _i, _vp, _i],
    "pcnn_learn": [_vp, _i, _i, C.POINTER(_f)],
    "pcnn_learn_host": [_vp, _vp, _i, _vp, _l, _i, _i, C.POINTER(_f)],
    "pcnn_err_sum": [_vp, C.POINTER(C.c_double), _i],
    "pcnn_forward_batch": [_vp, _vp, _i, _i, _vp, _vp],
    "pcnn_test": [_vp, C.POINTER(_l)],
    "pcnn_launch_count": [_vp, C.POINTER(_l)],
    "pcnn_step_errs": [_vp, _vp, _l, C.POINTER(_l)],
    "pcnn_time_fused_kernel": [_vp, _i, _i, C.POINTER(_f)],
    "pcnn_measure_fp32_peak": [_vp, C.POINTER(_f)],
    "pcnn_measure_tma_read": [_vp, _vp, _i, _i, _i, _i, _i, C.POINTER(_f)],
    "pcnn_measure_tma_write": [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, C.POINTER(_f)],
    "pcnn_measure_mma_rate": [_vp, _i, _i, _i, _i, _i, _i, C.POINTER(_f)],
    "pcnn_comm_unique_id": [_vp, C.POINTER(_sz)],
    "pcnn_comm_init_rank": [_vp, _vp, _i, _i],
    "pcnn_comm_destroy": [_vp],
    "pcnn_allreduce_grads": [_vp],
    "pcnn_p2p_export": [_vp, _vp, C.POINTER(_sz)],
    "pcnn_p2p_attach": [_vp, _vp, _i, _i],
    "pcnn_p2p_detach": [_vp],
    "pcnn_set_step_mode": [_vp, _i],
    "pcnn_persist_trace": [_vp, _vp, _i],
    "pcnn_persist_trace_ctas": [_vp, _vp, _i],
    "pcnn_persist_info": [_vp, _vp],
    "pcnn_conv_bwd_select": [_vp, _i],
    "pcnn_l5_compute_grads": [_vp, _vp, _vp, _i, _vp, _i, _vp],
    "pcnn_l5_train_step": [_vp, _vp, _vp, _i, _vp, _i, _vp],
    "pcnn_l5_forward": [_vp, _vp, _vp, _i, _i, _vp],
    "pcnn_persist_tune": [_vp, _i],
    "pcnn_maxpool_fwd": [_vp, _vp, _vp, _vp, _i, _i, _i, _i],
    "pcnn_maxpool_bwd": [_vp, _vp, _vp, _vp, _i, _i, _i, _i],
    "pcnn_softmax_ce": [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp],
    "pcnn_conv_tc_plan_create": [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _pvp],
    "pcnn_conv_tc_plan_create_strided": [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _pvp],
    "pcnn_conv_tc_plan_destroy": [_vp, _vp],
    "pcnn_conv_tc_plan_info": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_conv_tc_fwd": [_vp, _vp, _vp, _vp],
    "pcnn_conv_wide_plan_create": [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _pvp],
    "pcnn_conv_wide_plan_info": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_conv_wide_wgrad": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_conv_wide_dgrad": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_conv_wide_bwd_info": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_conv_wide_plan_create_padded": [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _pvp],
    "pcnn_conv_wide_plan_info_padded": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_conv_wide_wgrad_padded": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_conv_wide_dgrad_padded": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_conv_wide_bwd_info_padded": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_conv_wide_plan_create_dilated": [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _pvp],
    "pcnn_conv_wide_plan_info_dilated": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_conv_wide_wgrad_dilated": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_conv_wide_dgrad_dilated": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_conv_wide_bwd_info_dilated": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_f32_to_bf16_rows": [_vp, _vp, _vp, _l, _i, _i],
    "pcnn_conv_plan_set_params": [_vp, _vp, _vp, _vp],
    "pcnn_conv_bias_act_bwd": [_vp, _vp, _vp, _vp, _vp, _l, _i, _i],
    "pcnn_maxpool_nhwc_bf16_fwd": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_maxpool_nhwc_bf16_bwd": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_maxpool_nhwc_info": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_avgpool_nhwc_bf16_fwd": [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_avgpool_nhwc_bf16_bwd": [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_avgpool_nhwc_info": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_global_avgpool_nhwc_bf16_fwd": [_vp, _vp, _vp, _i, _i, _i, _i, _i],
    "pcnn_global_avgpool_nhwc_bf16_bwd": [_vp, _vp, _vp, _i, _i, _i, _i, _i],
    "pcnn_global_avgpool_nhwc_info": [_i, _i, _i, _i, _i, _vp],
    "pcnn_batchnorm_nhwc_bf16_fwd": [_vp, _vp, _vp, _vp, _l, _i, _i, _i, _f, _f, _vp, _vp, _vp, _vp, _vp, _vp],
    "pcnn_batchnorm_nhwc_bf16_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _l, _i, _i],
    "pcnn_batchnorm_nhwc_bf16_bwd_preact": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _l, _i, _i],
    "pcnn_batchnorm_nhwc_info": [_l, _i, _i, _vp],
    "pcnn_groupnorm_nhwc_bf16_fwd": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _vp, _vp, _vp],
    "pcnn_groupnorm_nhwc_bf16_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i],
    "pcnn_groupnorm_nhwc_bf16_bwd_preact": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i],
    "pcnn_groupnorm_nhwc_info": [_i, _i, _i, _i, _vp],
    "pcnn_attention_bf16_fwd": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _vp],
    "pcnn_attention_bf16_bwd": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _vp, _vp, _i],
    "pcnn_attention_info": [_i, _i, _i, _i, _i, _i, _f, _vp],
    "pcnn_conv_bwd_plan_info": [_i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_pad_nhwc_bf16": [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_crop_nhwc_bf16": [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_conv_wgrad": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_conv_dgrad": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_conv_wgrad_strided": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_conv_dgrad_strided": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i],
    "pcnn_conv_bwd_plan_info_strided": [_i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_linear_plan_create": [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _pvp],
    "pcnn_linear_wgrad": [_vp, _vp, _vp, _vp, _vp],
    "pcnn_linear_dgrad": [_vp, _vp, _vp, _vp],
    "pcnn_linear_info": [_i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_dwconv_plan_create": [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _pvp],
    "pcnn_dwconv_wgrad": [_vp, _vp, _vp, _vp, _vp],
    "pcnn_dwconv_dgrad": [_vp, _vp, _vp, _vp],
    "pcnn_dwconv_info": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_dwconv_plan_create_dilated": [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _pvp],
    "pcnn_dwconv_info_dilated": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_gconv_plan_create": [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _pvp],
    "pcnn_gconv_wgrad": [_vp, _vp, _vp, _vp, _vp],
    "pcnn_gconv_dgrad": [_vp, _vp, _vp, _vp],
    "pcnn_gconv_info": [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp],
    "pcnn_se_scale_nhwc_bf16_fwd": [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i],
    "pcnn_se_scale_nhwc_bf16_bwd_gate": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i],
    "pcnn_se_scale_nhwc_bf16_bwd_input": [_vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i],
    "pcnn_se_scale_nhwc_info": [_i, _i, _i, _i, _vp],
    "pcnn_dropout_bf16": [_vp, _vp, _vp, _vp, _i, _i, _i, C.c_double, _i, C.c_ulonglong, C.c_ulonglong],
    "pcnn_dropout_bf16_info": [_i, _i, _i, C.c_double, _i, _vp],
    "pcnn_augment_u8_bf16": [_vp, _vp, _vp, C.c_longlong, _i, _i, _i, C.c_longlong, _i, _i, _i, _i, C.c_ulonglong, C.c_ulonglong, _vp, _vp,
                             _vp, _i, _i, _i, _vp],
    "pcnn_augment_u8_bf16_info": [C.c_longlong, _i, _i, _i, C.c_longlong, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp],
    "pcnn_augment_mix_u8_bf16": [_vp, _vp, _vp, C.c_longlong, _i, _i, _i, C.c_longlong, _i, _i, _i, _i, C.c_ulonglong, C.c_ulonglong,
                                 _vp, _vp, _vp, _i, _i, _i, _vp, _i, C.c_double, _i, _i, _i, _i, _vp],
    "pcnn_augment_resized_u8_bf16": [_vp, _vp, _vp, C.c_longlong, _i, _i, _i, C.c_longlong, _i, _i, _i, C.c_ulonglong, C.c_ulonglong,
                                     _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _i, C.c_double, C.c_double, C.c_double, C.c_double, _i],
    "pcnn_augment_resized_u8_bf16_info": [C.c_longlong, _i, _i, _i, C.c_longlong, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _i,
                                          C.c_double, C.c_double, C.c_double, C.c_double, _i, _vp, _vp],
    "pcnn_augment_trivial_u8_bf16": [_vp, _vp, _vp, C.c_longlong, _i, _i, _i, C.c_longlong, _i, _i, _i, _i, C.c_ulonglong,
                                     C.c_ulonglong, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _i, _i] + [C.c_double] * 4 + [_i]
                                    + [C.c_double] * 5 + [_vp, C.c_longlong],
    "pcnn_augment_trivial_u8_bf16_info": [C.c_longlong, _i, _i, _i, C.c_longlong, _i, _i, _i, _i, _i, _i, _i] + [C.c_double] * 4
                                         + [_i] + [C.c_double] * 5 + [_i, _i, _i, _vp, _vp, _vp, _vp, _vp],
    "pcnn_softmax_ce_bf16": [_vp, _vp, _vp, _i, _i, _f, _vp, _vp, _vp],
    "pcnn_softmax_ce_soft_bf16": [_vp, _vp, _vp, _vp, C.c_double, C.c_double, _i, _i, _f, _vp, _vp, _vp],
    "pcnn_softmax_ce_pixels_bf16": [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp],
    "pcnn_conv_transpose_info": [_i] * 16 + [_vp],
    "pcnn_conv_transpose_fwd": [_vp, _vp, _vp, _vp, _vp] + [_i] * 15,
    "pcnn_upsample_bilinear_info": [_i] * 6 + [_vp],
    "pcnn_upsample_bilinear_nhwc_bf16_fwd": [_vp, _vp, _vp] + [_i] * 6,
    "pcnn_upsample_bilinear_nhwc_bf16_bwd": [_vp, _vp, _vp] + [_i] * 6,
    "pcnn_augment_mask_u8": [_vp, _vp, C.c_longlong, _i, _i, C.c_longlong, _i, _i, _i, _i, C.c_ulonglong, C.c_ulonglong, _i, _vp],
    "pcnn_pixel_shuffle_info": [_i] * 6 + [_vp],
    "pcnn_pixel_shuffle_nhwc_bf16": [_vp, _vp, _vp] + [_i] * 5,
    "pcnn_pixel_unshuffle_nhwc_bf16": [_vp, _vp, _vp] + [_i] * 5,
    "pcnn_regression_loss_bf16": [_vp, _vp, _vp, _i, _i, _i, _i, _f, _vp, _vp],
    "pcnn_gaussian_latent_info": [_i] * 4 + [_vp],
    "pcnn_gaussian_latent_bf16_fwd": [_vp, _vp, _i, _vp, _i, _vp, _i, _i, C.c_ulonglong, C.c_ulonglong, _i],
    "pcnn_gaussian_latent_bf16_bwd": [_vp, _vp, _i, _vp, _i, _vp, _i, _i, C.c_ulonglong, C.c_ulonglong, _f],
    "pcnn_bce_logits_bf16": [_vp, _vp, _vp, _i, _i, _i, _f, _vp, _vp],
    "pcnn_optim_create": [_vp, _vp, _vp, _i, _pvp],
    "pcnn_optim_step": [_vp, _vp, _f],
    "pcnn_optim_state": [_vp, _i, _pvp, _pvp],
    "pcnn_optim_info": [_vp, _vp],
    "pcnn_optim_destroy": [_vp, _vp],
}
_RESTYPE = {"pcnn_last_error_string": C.c_char_p, "pcnn_mnist_free": None}

_lib = None


def declared_symbols():
    """Every function name declared in include/pcnn.h (parsed from the header text)."""
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(pcnn_[a-z0-9_]+)\s*\(", text)))


def lib():
    """Load libpcnn.so (built in-tree by `make -C parallel-cnn_b200/csrc` / __graft_entry__.build()).  Fails loudly."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PcnnError("dlopen", -1, f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'`; "
                            "there is no CPU fallback")
        L = C.CDLL(LIB_PATH)
        for name, args in _SIG.items():
            fn = getattr(L, name)
            fn.argtypes = args
            fn.restype = _RESTYPE.get(name, C.c_int)
        _lib = L
    return _lib


def check(fn, code):
    if code != 0:
        raise PcnnError(fn, code, lib().pcnn_last_error_string().decode())


def init_params_reference():
    """The reference's static-constructor parameters (glibc rand(), seed 1) as a packed float32[2343] (host only)."""
    p = np.empty(NPARAM, np.float32)
    check("pcnn_init_params_reference", lib().pcnn_init_params_reference(p.ctypes.data))
    return p


def conv_tc_plan_info(N, H, W, C, K, R, S, stride=1, row_pitch=None, image_rows=0):
    """How the forward convolution plan tiles a shape (pcnn_conv_tc_plan_info; host only, no GPU).  row_pitch None = W*C
    rounded up to 8 elements, as ConvPlan."""
    pitch = (W * C + 7) // 8 * 8 if row_pitch is None else row_pitch
    out = (_i * 5)()
    check("pcnn_conv_tc_plan_info", lib().pcnn_conv_tc_plan_info(N, H, W, C, K, R, S, int(stride), int(pitch), int(image_rows), out))
    return dict(Qt=out[0], V=out[1], stages=out[2], n_mtiles=out[3], n_qtiles=out[4], tiles=out[3] * out[4])


def conv_wide_plan_info(N, H, W, C, K, R, S, stride=1, row_pitch=None, image_rows=0, padding=(0, 0), dilation=(1, 1)):
    """How the wide-channel forward plan tiles a shape (pcnn_conv_wide_plan_info, or pcnn_conv_wide_plan_info_padded for a
    padding (pad_h, pad_w) other than (0, 0), or pcnn_conv_wide_plan_info_dilated for a dilation (dil_h, dil_w) other than
    (1, 1); host only, no GPU).  row_pitch None = W*C rounded up to 8 elements, as WideConvPlan.  issued_pixels / useful_pixels:
    output pixels the tiles cover / compute."""
    pitch = (W * C + 7) // 8 * 8 if row_pitch is None else row_pitch
    ph, pw = (int(v) for v in padding)
    dh, dw = (int(v) for v in dilation)
    out = (_i * 8)()
    if (dh, dw) != (1, 1):
        check("pcnn_conv_wide_plan_info_dilated",
              lib().pcnn_conv_wide_plan_info_dilated(N, H, W, C, K, R, S, int(stride), ph, pw, dh, dw, int(pitch), int(image_rows), out))
    elif (ph, pw) == (0, 0):
        check("pcnn_conv_wide_plan_info", lib().pcnn_conv_wide_plan_info(N, H, W, C, K, R, S, int(stride), int(pitch), int(image_rows), out))
    else:
        check("pcnn_conv_wide_plan_info_padded",
              lib().pcnn_conv_wide_plan_info_padded(N, H, W, C, K, R, S, int(stride), ph, pw, int(pitch), int(image_rows), out))
    P, Q = (H + 2 * ph - dh * (R - 1) - 1) // stride + 1, (W + 2 * pw - dw * (S - 1) - 1) // stride + 1
    return dict(Pt=out[0], Qt=out[1], chunks=out[2], stages=out[3], tiles=out[4], n_pb=out[5], n_qb=out[6], npad=out[7],
                issued_pixels=out[4] * out[0] * out[1], useful_pixels=N * P * Q)


def conv_wide_bwd_info(N, H, W, C, K, R, S, stride=1, row_pitch=None, image_rows=0, padding=(0, 0), dilation=(1, 1)):
    """How the wide-channel gradients tile a shape (pcnn_conv_wide_bwd_info, or pcnn_conv_wide_bwd_info_padded for a padding
    (pad_h, pad_w) other than (0, 0), or pcnn_conv_wide_bwd_info_dilated for a dilation other than (1, 1); host only, no GPU).
    row_pitch None = W*C rounded up to 8 elements, as WideConvPlan.  wgrad_units = row-block pairs x pixel ranges;
    wgrad_blocks_per_split is the fewest."""
    pitch = (W * C + 7) // 8 * 8 if row_pitch is None else row_pitch
    ph, pw = (int(v) for v in padding)
    dh, dw = (int(v) for v in dilation)
    out = (_i * 10)()
    if (dh, dw) != (1, 1):
        check("pcnn_conv_wide_bwd_info_dilated",
              lib().pcnn_conv_wide_bwd_info_dilated(N, H, W, C, K, R, S, int(stride), ph, pw, dh, dw, int(pitch), int(image_rows), out))
    elif (ph, pw) == (0, 0):
        check("pcnn_conv_wide_bwd_info", lib().pcnn_conv_wide_bwd_info(N, H, W, C, K, R, S, int(stride), int(pitch), int(image_rows), out))
    else:
        check("pcnn_conv_wide_bwd_info_padded",
              lib().pcnn_conv_wide_bwd_info_padded(N, H, W, C, K, R, S, int(stride), ph, pw, int(pitch), int(image_rows), out))
    return dict(wgrad_row_blocks=out[0], wgrad_splits=out[1], wgrad_blocks_per_split=out[2], wgrad_stages=out[3], wgrad_units=out[4],
                dgrad_Pt=out[5], dgrad_Qt=out[6], dgrad_groups=out[7], dgrad_stages=out[8], dgrad_tiles=out[9])


def conv_transpose_info(N, H, W, C_in, C_out, R, S, stride=1, padding=(0, 0), output_padding=(0, 0), row_pitch=None, image_rows=0,
                        bias=False, act=0):
    """The output size, layout and input-gradient tiling of a transposed convolution (pcnn_conv_transpose_info; host only, no GPU),
    refused as pcnn_conv_transpose_fwd refuses.  row_pitch None = W_out * C_out (dense), image_rows 0 = H_out."""
    ph, pw = (int(v) for v in padding)
    oh, ow = (int(v) for v in output_padding)
    out = (_i * 8)()
    check("pcnn_conv_transpose_info", lib().pcnn_conv_transpose_info(int(N), int(H), int(W), int(C_in), int(C_out), int(R), int(S), int(stride),
                                                                     ph, pw, oh, ow, int(row_pitch or 0), int(image_rows), int(bool(bias)),
                                                                     int(act), out))
    return dict(H_out=out[0], W_out=out[1], row_pitch=out[2], image_rows=out[3], Pt=out[4], Qt=out[5], groups=out[6], tiles=out[7])


def upsample_bilinear_info(N, H, W, Cin, H_out, W_out):
    """How the bilinear resize partitions a shape (pcnn_upsample_bilinear_info; host only, no GPU), refused as its two passes
    refuse.  vec: channels per thread (8 or 1)."""
    out = (C.c_longlong * 4)()
    check("pcnn_upsample_bilinear_info", lib().pcnn_upsample_bilinear_info(int(N), int(H), int(W), int(Cin), int(H_out), int(W_out), out))
    return dict(vec=out[0], grid_fwd=out[1], grid_bwd=out[2], threads=out[3])


def pixel_shuffle_info(N, H, W, C, r, unshuffle=False):
    """How the pixel shuffle (unshuffle False: x [N][H][W][C r^2] -> [N][H r][W r][C]) or unshuffle (True: x [N][H][W][C] ->
    [N][H / r][W / r][C r^2]) partitions a shape (pcnn_pixel_shuffle_info; host only, no GPU), refused as the calls refuse.  vec:
    channels per thread (8 or 1); each CTA moves tile_pixels coarse pixels times chunk_channels fine channels through smem bytes."""
    out = (_ll * 6)()
    check("pcnn_pixel_shuffle_info", lib().pcnn_pixel_shuffle_info(int(N), int(H), int(W), int(C), int(r), int(bool(unshuffle)), out))
    return dict(vec=out[0], grid=out[1], threads=out[2], smem=out[3], tile_pixels=out[4], chunk_channels=out[5])


def gaussian_latent_info(R, L, ld=None, ldz=None):
    """How the Gaussian latent (stats [R][ld] -> z [R][ldz], ld None = 2L, ldz None = L) partitions a shape
    (pcnn_gaussian_latent_info; host only, no GPU), refused as the calls refuse.  vec: elements per thread (8 or 1); each CTA of
    threads takes tile_rows rows, chunk_columns columns per pass through smem bytes of KL terms."""
    out = (_ll * 6)()
    ld = 2 * int(L) if ld is None else int(ld)
    ldz = int(L) if ldz is None else int(ldz)
    check("pcnn_gaussian_latent_info", lib().pcnn_gaussian_latent_info(int(R), int(L), ld, ldz, out))
    return dict(vec=out[0], grid=out[1], threads=out[2], smem=out[3], tile_rows=out[4], chunk_columns=out[5])


def conv_layer_family(N, H, W, C, K, R, S, stride=1, padding=(0, 0), row_pitch=None, image_rows=0, dilation=(1, 1)):
    """Which forward plan serves a convolution layer (host only, no GPU): "narrow" (the row-Toeplitz plan,
    pcnn_conv_tc_plan_create_strided) when pcnn_conv_tc_plan_info accepts the shape and there is no padding, otherwise "wide"
    (pcnn_conv_wide_plan_create[_padded]).  The two domains do not overlap, so there is nothing to choose.  A padded shape the
    wide plan refuses but the row-Toeplitz plan takes unpadded (a narrow shape: few channels) has no padded kernel: it is
    refused with a PcnnError naming pcnn_pad_nhwc_bf16.  Any other shape neither plan takes gets the refusal of the plan its
    padding points to.  A dilation other than (1, 1) is "wide" (pcnn_conv_wide_plan_create_dilated) or that plan's refusal; with
    C % 8 != 0 it is refused with a PcnnError: no narrow-channel kernel dilates."""
    ph, pw = (int(v) for v in padding)
    dh, dw = (int(v) for v in dilation)
    if (dh, dw) != (1, 1):
        if C % 8 != 0:
            raise PcnnError("conv_layer_family", -1,
                            f"dilation ({dh}, {dw}) with C = {C} channels: no narrow-channel kernel dilates; only the wide plan "
                            "(C % 8 == 0) takes a dilation")
        conv_wide_plan_info(N, H, W, C, K, R, S, stride, row_pitch, image_rows, padding=(ph, pw), dilation=(dh, dw))
        return "wide"
    if (ph, pw) == (0, 0):
        try:
            conv_tc_plan_info(N, H, W, C, K, R, S, stride, row_pitch, image_rows)
            return "narrow"
        except PcnnError:
            conv_wide_plan_info(N, H, W, C, K, R, S, stride, row_pitch, image_rows)
            return "wide"
    try:
        conv_wide_plan_info(N, H, W, C, K, R, S, stride, row_pitch, image_rows, padding=(ph, pw))
        return "wide"
    except PcnnError as wide_refusal:
        try:
            conv_tc_plan_info(N, H, W, C, K, R, S, stride, row_pitch, image_rows)
        except PcnnError:
            raise wide_refusal
    raise PcnnError("conv_layer_family", -1,
                    f"padding ({ph}, {pw}) for a narrow shape (C = {C}, K = {K}, {R}x{S} taps) of the row-Toeplitz plan, which has no "
                    "padding: pad x into a zeroed canvas with pcnn_pad_nhwc_bf16 and build the layer on the canvas")


def maxpool_nhwc_info(N, H, W, C, R, S, stride, padding=(0, 0), row_pitch=0, image_rows=0):
    """The output size and layout of the NHWC max pool (pcnn_maxpool_nhwc_info; host only, no GPU).  row_pitch 0 = Q*C rounded up
    to 8 elements, image_rows 0 = P.  vec: channels per thread (8 or 1); cover: most windows over one input pixel."""
    ph, pw = (int(v) for v in padding)
    out = (_i * 5)()
    check("pcnn_maxpool_nhwc_info", lib().pcnn_maxpool_nhwc_info(int(N), int(H), int(W), int(C), int(R), int(S), int(stride), ph, pw,
                                                                 int(row_pitch), int(image_rows), out))
    return dict(P=out[0], Q=out[1], row_pitch=out[2], vec=out[3], cover=out[4])


def avgpool_nhwc_info(N, H, W, C, R, S, stride, padding=(0, 0), row_pitch=0, image_rows=0):
    """The output size and layout of the NHWC average pool (pcnn_avgpool_nhwc_info; host only, no GPU): the max pool's domain and
    keys (maxpool_nhwc_info)."""
    ph, pw = (int(v) for v in padding)
    out = (_i * 5)()
    check("pcnn_avgpool_nhwc_info", lib().pcnn_avgpool_nhwc_info(int(N), int(H), int(W), int(C), int(R), int(S), int(stride), ph, pw,
                                                                 int(row_pitch), int(image_rows), out))
    return dict(P=out[0], Q=out[1], row_pitch=out[2], vec=out[3], cover=out[4])


def global_avgpool_nhwc_info(N, H, W, C, row_pitch=0):
    """How the global average pool partitions a shape (pcnn_global_avgpool_nhwc_info; host only, no GPU).  row_pitch 0 = C rounded
    up to 8.  Lane l of a pixel range sums the pixels l, l + lanes, ... of it; the lanes, then the ranges, are added in order."""
    out = (_i * 8)()
    check("pcnn_global_avgpool_nhwc_info", lib().pcnn_global_avgpool_nhwc_info(int(N), int(H), int(W), int(C), int(row_pitch), out))
    return dict(row_pitch=out[0], vec=out[1], groups_per_cta=out[2], slices=out[3], lanes=out[4], pixels_per_cta=out[5], ranges=out[6],
                ctas=out[7])


def batchnorm_nhwc_info(pixels, C, training=True):
    """How batch normalization partitions dense [pixels][C] activations (pcnn_batchnorm_nhwc_info; host only, no GPU).  vec:
    channels per thread (8 or 1); lanes: pixels a CTA works on side by side; stat_slots (0 in eval) and grad_slots: per-CTA
    partials of the statistics and of the gradient pass, a function of (pixels, C) alone."""
    out = (_i * 5)()
    check("pcnn_batchnorm_nhwc_info", lib().pcnn_batchnorm_nhwc_info(int(pixels), int(C), 1 if training else 0, out))
    return dict(vec=out[0], lanes=out[1], pixels_per_cta=out[2], stat_slots=out[3], grad_slots=out[4])


def groupnorm_nhwc_info(N, HW, C, G):
    """How group normalization partitions dense [N][HW][C] activations in G groups (pcnn_groupnorm_nhwc_info; host only, no GPU),
    refused as the entry points refuse.  vec: channels per thread (8 or 1); the C / vec channel groups are cut into `slices` of
    `groups_per_cta`, each image's HW pixels into `ranges` of `pixels_per_range` (both a function of (HW, C, G) alone); ctas: the
    grid of every elementwise pass; slots: per-CTA partials per channel (N * ranges); group_ctas: the grid of the per-(n, g) merges;
    n_acc (dgamma, dbeta) and n_acc_group (A, B, the statistics): fp32 roundings on the longest path of one sum."""
    out = (_i * 11)()
    check("pcnn_groupnorm_nhwc_info", lib().pcnn_groupnorm_nhwc_info(int(N), int(HW), int(C), int(G), out))
    return dict(vec=out[0], groups_per_cta=out[1], slices=out[2], lanes=out[3], pixels_per_range=out[4], ranges=out[5], ctas=out[6],
                slots=out[7], group_ctas=out[8], n_acc=out[9], n_acc_group=out[10])


def attention_info(N, T, heads, d, ld=None, ld_g=0, scale=None):
    """How self-attention tiles a shape (pcnn_attention_info; host only, no GPU), refused as the device calls refuse.  ld None =
    heads * d (separate dense q, k and v); ld_g 0 leaves out the backward's output rule; scale None = 1 / sqrt(d)."""
    ld = int(heads) * int(d) if ld is None else int(ld)
    scale = 1.0 / math.sqrt(d) if scale is None else float(scale)
    out = (_ll * 8)()
    check("pcnn_attention_info", lib().pcnn_attention_info(int(N), int(T), int(heads), int(d), ld, int(ld_g), scale, out))
    return dict(query_rows=out[0], block_rows=out[1], stages=out[2], fwd_tiles=out[3], dkdv_tiles=out[4], dq_tiles=out[5],
                scratch_bytes=out[6], bwd_smem=out[7])


def linear_info(N, P, Q, C, O, row_pitch=0, image_rows=0):
    """How the fully connected layer tiles a shape (pcnn_linear_info; host only, no GPU).  row_pitch 0 = Q*C rounded up to 8
    elements, image_rows 0 = P.  Each pass splits its reduction as a function of the shape alone."""
    out = (_i * 12)()
    check("pcnn_linear_info", lib().pcnn_linear_info(int(N), int(P), int(Q), int(C), int(O), int(row_pitch), int(image_rows), out))
    return dict(row_pitch=out[0], image_tiles=out[1], fwd_steps=out[2], fwd_splits=out[3], fwd_stages=out[4], wgrad_pairs=out[5],
                wgrad_splits=out[6], wgrad_stages=out[7], dgrad_tiles=out[8], dgrad_chunks=out[9], dgrad_stages=out[10], npad=out[11])


def dwconv_info(N, H, W, C, R, S, stride=1, padding=(0, 0), dilation=(1, 1)):
    """The output size and the weight-gradient split of the depthwise convolution (pcnn_dwconv_info, or pcnn_dwconv_info_dilated
    for a dilation other than (1, 1); host only, no GPU), refused as the create call refuses.  vec: channels per thread (8 or 1);
    the N*P*Q output pixels are cut into `ranges` of `pixels_per_range`, a function of the shape alone; n_acc: fp32 additions on
    the longest path of one dw sum."""
    ph, pw = (int(v) for v in padding)
    dh, dw = (int(v) for v in dilation)
    out = (_i * 9)()
    if (dh, dw) != (1, 1):
        check("pcnn_dwconv_info_dilated", lib().pcnn_dwconv_info_dilated(int(N), int(H), int(W), int(C), int(R), int(S), int(stride), ph, pw,
                                                                       dh, dw, out))
    else:
        check("pcnn_dwconv_info", lib().pcnn_dwconv_info(int(N), int(H), int(W), int(C), int(R), int(S), int(stride), ph, pw, out))
    return dict(P=out[0], Q=out[1], vec=out[2], groups_per_cta=out[3], slices=out[4], lanes=out[5], pixels_per_range=out[6],
                ranges=out[7], n_acc=out[8])


def gconv_info(N, H, W, C, K, G, R, S, stride=1, padding=(0, 0)):
    """The output size, the tiling and the weight-gradient split of the grouped convolution (pcnn_gconv_info; host only, no GPU),
    refused as pcnn_gconv_plan_create refuses.  vec: x channels per load (8, 4, 2 or 1, the largest dividing Cg; 8 is the 16-byte
    path); kt: output channels per forward thread and dy channels per input-gradient load (the largest dividing Kg); the N*P*Q
    output pixels are cut into `ranges` of `pixels_per_range`, a function of the shape alone; n_acc: fp32 additions on the longest
    path of one dw sum."""
    ph, pw = (int(v) for v in padding)
    out = (_i * 16)()
    check("pcnn_gconv_info", lib().pcnn_gconv_info(int(N), int(H), int(W), int(C), int(K), int(G), int(R), int(S), int(stride), ph, pw,
                                                   out))
    return dict(P=out[0], Q=out[1], Cg=out[2], Kg=out[3], vec=out[4], kt=out[5], fwd_tiles_per_cta=out[6], fwd_slices=out[7],
                dgrad_tiles_per_cta=out[8], dgrad_slices=out[9], wgrad_items=out[10], wgrad_item_blocks=out[11], pixels_per_range=out[12],
                ranges=out[13], n_acc=out[14], lanes=out[15])


def se_scale_nhwc_info(N, H, W, C):
    """How the squeeze-and-excitation gate gradient partitions a shape (pcnn_se_scale_nhwc_info; host only, no GPU): the global
    average pool's partition (global_avgpool_nhwc_info), refused as the three passes refuse.  vec: channels per thread (8 or 1);
    n_acc: fp32 additions on the longest path of one ds sum."""
    out = (_i * 8)()
    check("pcnn_se_scale_nhwc_info", lib().pcnn_se_scale_nhwc_info(int(N), int(H), int(W), int(C), out))
    return dict(vec=out[0], groups_per_cta=out[1], slices=out[2], lanes=out[3], pixels_per_cta=out[4], ranges=out[5], ctas=out[6],
                n_acc=out[7])


def dropout_info(N, row_elems, row_pitch=0, p=0.0, per_sample=False):
    """The mask rule and the launch of the dropout kernel (pcnn_dropout_bf16_info; host only, no GPU), refused as pcnn_dropout_bf16
    refuses.  row_pitch 0 = dense.  T: an element is dropped iff its Philox draw < T; scale_bits: the fp32 bits of 1 / (1 - p);
    vec: elements per vector (8 is the 16-byte path); grid: CTAs of 256 threads; per_thread: elements of the busiest thread."""
    out = (C.c_longlong * 5)()
    check("pcnn_dropout_bf16_info", lib().pcnn_dropout_bf16_info(int(N), int(row_elems), int(row_pitch), float(p), int(per_sample), out))
    return dict(T=out[0], scale_bits=out[1], vec=out[2], grid=out[3], per_thread=out[4])


def channel_stats(values, C, name):
    """mean or std of the input pipeline as a float32 array of C values (None stays None: mean 0 / std 1); a scalar is every channel's"""
    if values is None:
        return None
    a = np.asarray(values, np.float32).reshape(-1)
    if np.ndim(values) == 0:
        a = np.repeat(a, int(C))
    if a.size != int(C):
        raise PcnnError("augment", -1, f"{name} has {a.size} values for C = {C} channels")
    return a


def augment_info(n, H, W, C, first, N, shuffle=1, pad=0, flip=0, C_out=None, row_pitch=0, image_rows=0, mean=None, std=None):
    """The layout, permutation width, launch and value table of the input pipeline (pcnn_augment_u8_bf16_info; host only, no GPU),
    refused as pcnn_augment_u8_bf16 refuses.  C_out None = C; row_pitch / image_rows 0 = dense; mean / std None = 0 / 1.
    Returns (info, lut): info holds row_pitch and image_rows as used, b (the Feistel half width), vec (elements per vector, 8 is the
    16-byte path), grid, rows_per_cta, row_blocks (per image) and threads; lut is uint16 [C][256], the bf16 bits of each value."""
    Cin = int(C)
    C_out = Cin if C_out is None else int(C_out)
    m, s = channel_stats(mean, Cin, "mean"), channel_stats(std, Cin, "std")
    out = (_ll * 8)()
    lut = np.zeros((max(Cin, 1), 256), np.uint16)
    check("pcnn_augment_u8_bf16_info", lib().pcnn_augment_u8_bf16_info(
        int(n), int(H), int(W), Cin, int(first), int(N), int(shuffle), int(pad), int(flip), C_out, int(row_pitch or 0),
        int(image_rows or 0), None if m is None else m.ctypes.data, None if s is None else s.ctypes.data, out,
        lut.ctypes.data if 1 <= Cin <= 4 else None))
    keys = ("row_pitch", "image_rows", "b", "vec", "grid", "rows_per_cta", "row_blocks", "threads")
    return dict(zip(keys, list(out))), lut


RESIZE_TRAIN, RESIZE_EVAL = 1, 2        # pcnn_augment_resized_u8_bf16's modes


def augment_resized_info(n, H, W, C, first, N, H_out, W_out, mode=RESIZE_TRAIN, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3), resize_size=0,
                         shuffle=1, flip=0, C_out=None, row_pitch=0, image_rows=0, mean=None, std=None):
    """The layout, launch, resized size, window, fallback box and value table of a resized batch (pcnn_augment_resized_u8_bf16_info;
    host only, no GPU), refused as pcnn_augment_resized_u8_bf16 refuses.  Returns (info, lut): info holds augment_info's keys plus
    smem (dynamic shared bytes per CTA), taps_y, taps_x, rows_cap, Rh, Rw (the resized image), ty, tx (the window's offset in it)
    fallback (top, left, height, width) and static_smem (the kernel's static shared bytes; smem + static_smem <= 48 KB)."""
    Cin = int(C)
    C_out = Cin if C_out is None else int(C_out)
    m, s = channel_stats(mean, Cin, "mean"), channel_stats(std, Cin, "std")
    out = (_ll * 21)()
    lut = np.zeros((max(Cin, 1), 256), np.uint16)
    check("pcnn_augment_resized_u8_bf16_info", lib().pcnn_augment_resized_u8_bf16_info(
        int(n), int(H), int(W), Cin, int(first), int(N), int(shuffle), int(flip), int(H_out), int(W_out), C_out, int(row_pitch or 0),
        int(image_rows or 0), None if m is None else m.ctypes.data, None if s is None else s.ctypes.data, int(mode), float(scale[0]),
        float(scale[1]), float(ratio[0]), float(ratio[1]), int(resize_size or 0), out, lut.ctypes.data if 1 <= Cin <= 4 else None))
    keys = ("row_pitch", "image_rows", "b", "vec", "grid", "rows_per_cta", "row_blocks", "threads", "smem", "taps_y", "taps_x",
            "rows_cap", "Rh", "Rw", "ty", "tx")
    info = dict(zip(keys, list(out)[:16]))
    info["fallback"] = tuple(out[16:20])
    info["static_smem"] = out[20]
    return info, lut


TRIVIAL_NONE, TRIVIAL_NEAREST, TRIVIAL_BILINEAR = 0, 1, 2       # pcnn_augment_trivial_u8_bf16's interpolations
TRIVIAL_OPS = ("Identity", "ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate", "Brightness", "Color", "Contrast", "Sharpness",
               "Posterize", "Solarize", "AutoContrast", "Equalize")


def augment_trivial_info(n, H, W, C, first, N, trivial=TRIVIAL_NEAREST, erase_p=0.0, erase_scale=(0.02, 0.33), erase_ratio=(0.3, 3.3),
                         crop_size=None, scale=(0.08, 1.0), ratio=(3 / 4, 4 / 3), shuffle=1, pad=0, flip=0, C_out=None, row_pitch=0,
                         image_rows=0, mean=None, std=None):
    """The layout, workspace, launch, magnitude table and value table of a TrivialAugmentWide / RandomErasing batch
    (pcnn_augment_trivial_u8_bf16_info; host only, no GPU), refused as pcnn_augment_trivial_u8_bf16 refuses.  crop_size None is the
    plain geometry (pad, flip), (h, w) the resized call's RandomResizedCrop.  Returns (info, table, lut): info holds row_pitch,
    image_rows, h, w, ws_pitch, ws_bytes, vec, grid, threads, smem, static_smem and arg_bytes; table float32 [14][31][2][6]."""
    Cin = int(C)
    C_out = Cin if C_out is None else int(C_out)
    m, s = channel_stats(mean, Cin, "mean"), channel_stats(std, Cin, "std")
    out = (_ll * 12)()
    table = np.zeros((14, 31, 2, 6), np.float32)
    lut = np.zeros((max(Cin, 1), 256), np.uint16)
    hw = (0, 0) if crop_size is None else tuple(int(v) for v in crop_size)
    check("pcnn_augment_trivial_u8_bf16_info", lib().pcnn_augment_trivial_u8_bf16_info(
        int(n), int(H), int(W), Cin, int(first), int(N), int(shuffle), int(pad), int(flip), int(crop_size is not None), *hw,
        float(scale[0]), float(scale[1]), float(ratio[0]), float(ratio[1]), int(trivial), float(erase_p), float(erase_scale[0]),
        float(erase_scale[1]), float(erase_ratio[0]), float(erase_ratio[1]), C_out, int(row_pitch or 0), int(image_rows or 0),
        None if m is None else m.ctypes.data, None if s is None else s.ctypes.data, out, table.ctypes.data,
        lut.ctypes.data if 1 <= Cin <= 4 else None))
    keys = ("row_pitch", "image_rows", "h", "w", "ws_pitch", "ws_bytes", "vec", "grid", "threads", "smem", "static_smem", "arg_bytes")
    return dict(zip(keys, list(out))), table, lut


def conv_bwd_plan_info(N, H, W, C, K, R, S, stride=1):
    """Which kernels the backward passes pick for a shape and how they tile it (pcnn_conv_bwd_plan_info_strided; host only,
    no GPU).  dgrad_ring: partial dx rows each consumer thread keeps in registers."""
    out = (_i * 9)()
    check("pcnn_conv_bwd_plan_info_strided", lib().pcnn_conv_bwd_plan_info_strided(N, H, W, C, K, R, S, int(stride), out))
    return dict(wgrad_tc=bool(out[0]), wgrad_rb=out[1], wgrad_pc=out[2], wgrad_stages=out[3],
                dgrad_tc=bool(out[4]), dgrad_strips=out[5], dgrad_oq=out[6], dgrad_ring=out[7], dgrad_stages=out[8])


def mnist_load_u8(image_file, label_file):
    """mnist_load's contract (return codes 0, -1..-4) on raw u8; returns (code, images[n,784] u8, labels[n] u8)."""
    L = lib()
    img, lab, cnt = C.c_void_p(), C.c_void_p(), C.c_uint(0)
    rc = L.pcnn_mnist_load_u8(os.fsencode(image_file), os.fsencode(label_file), C.byref(img), C.byref(lab), C.byref(cnt))
    if rc != 0:
        return rc, None, None
    n = cnt.value
    images = np.ctypeslib.as_array(C.cast(img, C.POINTER(C.c_uint8)), shape=(n * 784,)).reshape(n, 784).copy()
    labels = np.ctypeslib.as_array(C.cast(lab, C.POINTER(C.c_uint8)), shape=(n,)).copy()
    L.pcnn_mnist_free(img)
    L.pcnn_mnist_free(lab)
    return 0, images, labels
