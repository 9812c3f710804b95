"""parallel-cnn_b200 -- Python host mirror of the libpcnn.so C ABI (include/pcnn.h).

The product is the CUDA library built from csrc/ (hand-written sm_90a kernels behind a plain C ABI that replaces
/root/reference/Sequential/layer.h + Main.cpp for the LeNet/MNIST training path).  This module only binds that ABI
with ctypes so tests, bench.py and __graft_entry__ can drive it; it carries NO compute of its own and NO CPU
fallback: if libpcnn.so is missing or no sm_90 GPU is present, every compute entry point raises.

The directory name contains a hyphen, so import it through ``pcnn_loader.load()`` at the repo root (which registers
it as the module ``parallel_cnn_b200``).
"""
from ._lib import (  # noqa: F401
    LIB_PATH, NPARAM, OFF, PcnnError, U8, F32, TRAIN_SET, TEST_SET, MODE_AUTO, MODE_GRAPH, MODE_PERSISTENT,
    lib, declared_symbols, init_params_reference, mnist_load_u8,
)
from .engine import ConvPlan, DeviceArray, Engine, bf16_bits_to_f32, f32_to_bf16_bits  # noqa: F401

__all__ = ["Engine", "DeviceArray", "PcnnError", "lib", "declared_symbols", "init_params_reference",
           "mnist_load_u8", "NPARAM", "OFF", "U8", "F32", "TRAIN_SET", "TEST_SET", "LIB_PATH"]
