"""parallel-cnn_b200 -- Python host mirror of the libpcnn.so C ABI (include/pcnn.h).

The product is the CUDA library built from csrc/ (hand-written sm_90a kernels behind a plain C ABI that replaces
/root/reference/Sequential/layer.h + Main.cpp for the LeNet/MNIST training path).  This module only binds that ABI
with ctypes so tests, bench.py and __graft_entry__ can drive it; it carries NO compute of its own and NO CPU
fallback: if libpcnn.so is missing or no sm_90 GPU is present, every compute entry point raises.

The directory name contains a hyphen, so import it through ``pcnn_loader.load()`` at the repo root (which registers
it as the module ``parallel_cnn_b200``).
"""
from ._lib import (  # noqa: F401
    LIB_PATH, NPARAM, OFF, PcnnError, U8, F32, TRAIN_SET, TEST_SET, MODE_AUTO, MODE_GRAPH, MODE_PERSISTENT, ACT_NONE, ACT_SIGMOID, ACT_RELU,
    ACT_SILU, ACT_HARDSWISH, ACT_RELU6,
    lib, declared_symbols, init_params_reference, mnist_load_u8, conv_tc_plan_info, conv_wide_plan_info, conv_wide_bwd_info,
    conv_bwd_plan_info, conv_layer_family, maxpool_nhwc_info, avgpool_nhwc_info, global_avgpool_nhwc_info, batchnorm_nhwc_info,
    groupnorm_nhwc_info, attention_info,
    linear_info, dwconv_info, gconv_info, se_scale_nhwc_info, dropout_info, augment_info, augment_resized_info, RESIZE_TRAIN, RESIZE_EVAL, OPTIM_SGD, OPTIM_ADAMW,
    augment_trivial_info, TRIVIAL_NONE, TRIVIAL_NEAREST, TRIVIAL_BILINEAR, TRIVIAL_OPS, conv_transpose_info, upsample_bilinear_info,
    pixel_shuffle_info, LOSS_MSE, LOSS_L1, gaussian_latent_info,
)
from .engine import AvgPoolLayer, BatchNormLayer, GroupNormLayer, ConvLayer, GlobalAvgPoolLayer, ConvPlan, LinearLayer, LinearPlan, MaxPoolLayer, DeviceArray, WideConvPlan, Engine, bf16_bits_to_f32, f32_to_bf16_bits  # noqa: F401
from .engine import DepthwiseConvLayer, DepthwiseConvPlan, DropoutLayer, GroupedConvLayer, GroupedConvPlan, SqueezeExcitationLayer  # noqa: F401
from .engine import ImageBatcher, MixedLabels, MIX_MIXUP, MIX_CUTMIX, mix_draws  # noqa: F401
from .engine import SGD, AdamW, FusedOptimizer  # noqa: F401
from .engine import ConvTransposeLayer, UpsampleBilinearLayer, segmentation_scores  # noqa: F401
from .engine import SelfAttentionLayer  # noqa: F401
from .engine import PixelShuffleLayer, PixelUnshuffleLayer, psnr  # noqa: F401
from .engine import GaussianLatentLayer  # noqa: F401

__all__ = ["Engine", "DeviceArray", "PcnnError", "lib", "declared_symbols", "init_params_reference",
           "mnist_load_u8", "conv_tc_plan_info", "conv_wide_plan_info", "conv_wide_bwd_info", "conv_bwd_plan_info", "conv_layer_family", "maxpool_nhwc_info", "avgpool_nhwc_info", "global_avgpool_nhwc_info", "batchnorm_nhwc_info", "linear_info", "ConvLayer", "BatchNormLayer", "MaxPoolLayer", "AvgPoolLayer", "GlobalAvgPoolLayer", "LinearLayer", "ConvPlan", "LinearPlan",
           "WideConvPlan", "NPARAM", "OFF", "U8", "F32", "TRAIN_SET", "TEST_SET", "LIB_PATH", "ACT_NONE", "ACT_SIGMOID", "ACT_RELU",
           "ACT_SILU", "ACT_HARDSWISH", "ACT_RELU6",
           "SGD", "AdamW", "FusedOptimizer", "OPTIM_SGD", "OPTIM_ADAMW", "dwconv_info", "DepthwiseConvLayer", "DepthwiseConvPlan",
           "gconv_info", "GroupedConvLayer", "GroupedConvPlan", "se_scale_nhwc_info", "SqueezeExcitationLayer",
           "dropout_info", "DropoutLayer", "augment_info", "augment_resized_info", "RESIZE_TRAIN", "RESIZE_EVAL", "ImageBatcher",
           "MixedLabels", "MIX_MIXUP", "MIX_CUTMIX", "mix_draws", "augment_trivial_info", "TRIVIAL_NONE", "TRIVIAL_NEAREST",
           "TRIVIAL_BILINEAR", "TRIVIAL_OPS", "conv_transpose_info", "upsample_bilinear_info", "ConvTransposeLayer",
           "UpsampleBilinearLayer", "segmentation_scores", "groupnorm_nhwc_info", "GroupNormLayer", "attention_info", "SelfAttentionLayer",
           "pixel_shuffle_info", "LOSS_MSE", "LOSS_L1", "PixelShuffleLayer", "PixelUnshuffleLayer", "psnr",
           "gaussian_latent_info", "GaussianLatentLayer"]
