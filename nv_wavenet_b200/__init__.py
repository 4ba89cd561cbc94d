"""nv_wavenet_b200 -- H100-native (sm_90a) autoregressive WaveNet inference behind nv-wavenet's interfaces.

The package is only the host-side mirror of the reference's operator interface; every computation
runs in nv_wavenet_b200/lib/libwavenet_infer.so (hand-written CUDA, C-ABI in include/*.h).
"""
from ._lib import FP16, FP32, FP32_FAST, KERNEL_AUTO, KERNEL_LATENCY, KERNEL_STREAM, KERNEL_TENSORCORE, LIB_PATH, NvwnError  # noqa: F401
from .infer import (AUTO, DUAL_BLOCK, MANYBLOCK_NONPERSISTENT, PERSISTENT, SINGLE_BLOCK,  # noqa: F401
                    NVWavenetInfer)
