"""neuralampmodelercore_b200 -- NeuralAmpModelerCore's per-sample inference hot path, H100-native (sm_90a).

The package holds only what the path needs: csrc/ (hand-written sm_90a kernels + the C ABI of
include/nam_b200.h, built in-tree into lib/libnam_b200.so) and a thin Python mirror of the reference's
nam::DSP / nam::get_dsp interface (dsp.py) used by tests and bench.py.
"""
from ._build import build, LIB_PATH  # noqa: F401
from .dsp import (  # noqa: F401
    DSP,
    bank_check,
    bank_jit_prepare,
    CudaUnavailableError,
    NamFileValidationError,
    UnsupportedModelError,
    disable_fast_tanh,
    enable_fast_tanh,
    get_dsp,
    get_dsp_bank,
    inspect,
    jit_prepare,
    measure_fp32_tflops,
    has_tensor_core_kernel,
    resampler,
    state_layout,
    submodels,
    using_fast_tanh,
)

__all__ = [
    "build",
    "LIB_PATH",
    "DSP",
    "get_dsp",
    "get_dsp_bank",
    "bank_check",
    "bank_jit_prepare",
    "inspect",
    "jit_prepare",
    "submodels",
    "state_layout",
    "resampler",
    "enable_fast_tanh",
    "disable_fast_tanh",
    "using_fast_tanh",
    "measure_fp32_tflops",
    "has_tensor_core_kernel",
    "NamFileValidationError",
    "UnsupportedModelError",
    "CudaUnavailableError",
]
