"""ctypes declarations for include/nam_b200.h (the C ABI of libnam_b200.so)."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

from . import _build

_lib = None

f32p = C.POINTER(C.c_float)
f64p = C.POINTER(C.c_double)


class _OptionsWords(C.Structure):
    _fields_ = [("resample", C.c_int32), ("reserved_tail", C.c_int32 * 3)]


class _OptionsTail(C.Union):
    _anonymous_ = ("_words",)
    _fields_ = [("reserved", C.c_int32 * 4), ("_words", _OptionsWords)]


class Options(C.Structure):
    _anonymous_ = ("_tail",)
    _fields_ = [
        ("struct_size", C.c_int32),
        ("device", C.c_int32),
        ("max_batch", C.c_int32),
        ("fast_tanh", C.c_int32),
        ("prewarm_on_reset", C.c_int32),
        ("ctas_per_sm", C.c_int32),
        ("kernel_geometry", C.c_int32),
        ("tile_mode", C.c_int32),
        ("jit", C.c_int32),
        ("bank_capacity", C.c_int32),
        ("_tail", _OptionsTail),
    ]


class Info(C.Structure):
    _fields_ = [
        ("struct_size", C.c_int32),
        ("architecture", C.c_int32),
        ("in_channels", C.c_int32),
        ("out_channels", C.c_int32),
        ("prewarm_samples", C.c_int32),
        ("max_batch", C.c_int32),
        ("max_frames", C.c_int32),
        ("has_loudness", C.c_int32),
        ("has_input_level", C.c_int32),
        ("has_output_level", C.c_int32),
        ("expected_sample_rate", C.c_double),
        ("loudness", C.c_double),
        ("input_level_dbu", C.c_double),
        ("output_level_dbu", C.c_double),
        ("n_weights", C.c_int64),
        ("state_bytes_per_stream", C.c_int64),
        ("flops_per_frame", C.c_double),
        ("kernel_variant", C.c_int32),
        ("jit_state", C.c_int32),
        ("jit_lat_state", C.c_int32),
        ("resample_up", C.c_int32),
        ("resample_down", C.c_int32),
        ("resample_latency_frames", C.c_int32),
        ("reserved", C.c_int32 * 2),
    ]


# Every symbol include/nam_b200.h declares; tests check the built library exports all of them.
EXPORTED_SYMBOLS = [
    "nam_b200_default_options",
    "nam_b200_abi_version",
    "nam_b200_create_from_file",
    "nam_b200_create_from_json",
    "nam_b200_destroy",
    "nam_b200_get_info",
    "nam_b200_reset",
    "nam_b200_prewarm",
    "nam_b200_process_f32",
    "nam_b200_process_f32_device",
    "nam_b200_process_f64_planar",
    "nam_b200_process_f32_planar",
    "nam_b200_set_fast_tanh",
    "nam_b200_set_reserved_sms",
    "nam_b200_has_tensor_core_kernel",
    "nam_b200_set_slimmable_size",
    "nam_b200_slimmable_breakpoints",
    "nam_b200_synchronize",
    "nam_b200_launch_count",
    "nam_b200_last_kernel_ms",
    "nam_b200_last_error",
    "nam_b200_measure_fp32_tflops",
    "nam_b200_inspect_json",
    "nam_b200_inspect_file",
    "nam_b200_submodel_json",
    "nam_b200_jit_prepare_json",
    "nam_b200_jit_prepare_json_for_batch",
    "nam_b200_jit_note",
    "nam_b200_pin_host_buffer",
    "nam_b200_unpin_host_buffer",
    "nam_b200_host_buffer_is_pinned",
    "nam_b200_multi_create_from_file",
    "nam_b200_multi_create_from_json",
    "nam_b200_multi_destroy",
    "nam_b200_multi_device_count",
    "nam_b200_multi_shard",
    "nam_b200_multi_reset",
    "nam_b200_multi_process_f32",
    "nam_b200_stream_state_size",
    "nam_b200_reset_streams",
    "nam_b200_copy_streams",
    "nam_b200_export_streams",
    "nam_b200_import_streams",
    "nam_b200_export_streams_device",
    "nam_b200_import_streams_device",
    "nam_b200_state_layout_json",
    "nam_b200_process_streams_f32",
    "nam_b200_process_streams_f32_device",
    "nam_b200_process_streams_ragged_f32",
    "nam_b200_process_streams_ragged_f32_device",
    "nam_b200_create_bank_from_json",
    "nam_b200_create_bank_from_files",
    "nam_b200_bank_size",
    "nam_b200_assign_streams",
    "nam_b200_stream_models",
    "nam_b200_bank_model_info",
    "nam_b200_bank_check_json",
    "nam_b200_bank_jit_prepare_json",
    "nam_b200_bank_capacity",
    "nam_b200_bank_add_models",
    "nam_b200_bank_replace_model",
    "nam_b200_resampler_json",
]


def lib_path() -> Path:
    return _build.LIB_PATH


def load(build_if_missing: bool = True) -> C.CDLL:
    """Load libnam_b200.so.  Fails loudly (RuntimeError) if the CUDA extension is absent: there is no
    Python or CPU fallback for the hot path."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB_PATH
    if not path.exists():
        if not build_if_missing:
            raise RuntimeError(f"{path} is missing: build it with neuralampmodelercore_b200.build()")
        _build.build()
    try:
        lib = C.CDLL(str(path))
    except OSError as e:
        raise RuntimeError(f"could not load the CUDA extension {path}: {e}") from e
    vp = C.c_void_p
    lib.nam_b200_default_options.argtypes = [C.POINTER(Options)]
    lib.nam_b200_default_options.restype = None
    lib.nam_b200_abi_version.restype = C.c_int
    lib.nam_b200_create_from_file.argtypes = [C.c_char_p, C.POINTER(Options), C.POINTER(vp)]
    lib.nam_b200_create_from_json.argtypes = [C.c_char_p, C.POINTER(Options), C.POINTER(vp)]
    lib.nam_b200_destroy.argtypes = [vp]
    lib.nam_b200_destroy.restype = None
    lib.nam_b200_get_info.argtypes = [vp, C.POINTER(Info)]
    lib.nam_b200_reset.argtypes = [vp, C.c_double, C.c_int]
    lib.nam_b200_prewarm.argtypes = [vp]
    lib.nam_b200_process_f32.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int64, C.c_int64]
    lib.nam_b200_process_f32_device.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int64, C.c_int64, vp]
    lib.nam_b200_process_f64_planar.argtypes = [vp, C.POINTER(f64p), C.POINTER(f64p), C.c_int]
    lib.nam_b200_process_f32_planar.argtypes = [vp, C.POINTER(f32p), C.POINTER(f32p), C.c_int]
    lib.nam_b200_set_fast_tanh.argtypes = [vp, C.c_int]
    lib.nam_b200_set_reserved_sms.argtypes = [vp, C.c_int]
    lib.nam_b200_set_slimmable_size.argtypes = [vp, C.c_double]
    lib.nam_b200_slimmable_breakpoints.argtypes = [vp, C.POINTER(C.c_double), C.c_int]
    lib.nam_b200_synchronize.argtypes = [vp]
    lib.nam_b200_launch_count.argtypes = [vp]
    lib.nam_b200_launch_count.restype = C.c_int64
    lib.nam_b200_last_kernel_ms.argtypes = [vp]
    lib.nam_b200_last_kernel_ms.restype = C.c_double
    lib.nam_b200_last_error.restype = C.c_char_p
    lib.nam_b200_inspect_json.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int64]
    lib.nam_b200_inspect_json.restype = C.c_int
    lib.nam_b200_inspect_file.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int64]
    lib.nam_b200_inspect_file.restype = C.c_int
    lib.nam_b200_submodel_json.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_double), C.c_char_p, C.c_int64]
    lib.nam_b200_submodel_json.restype = C.c_int64
    lib.nam_b200_jit_prepare_json.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int64]
    lib.nam_b200_jit_prepare_json.restype = C.c_int
    lib.nam_b200_jit_prepare_json_for_batch.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_char_p, C.c_int64]
    lib.nam_b200_jit_prepare_json_for_batch.restype = C.c_int
    lib.nam_b200_jit_note.argtypes = [C.c_void_p, C.c_char_p, C.c_int64]
    lib.nam_b200_jit_note.restype = C.c_int64
    lib.nam_b200_pin_host_buffer.argtypes = [C.c_void_p, C.c_int64]
    lib.nam_b200_unpin_host_buffer.argtypes = [C.c_void_p]
    lib.nam_b200_host_buffer_is_pinned.argtypes = [C.c_void_p]
    lib.nam_b200_multi_create_from_json.argtypes = [C.c_char_p, C.c_void_p, C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_void_p)]
    lib.nam_b200_multi_create_from_file.argtypes = [C.c_char_p, C.c_void_p, C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_void_p)]
    lib.nam_b200_multi_destroy.argtypes = [C.c_void_p]
    lib.nam_b200_multi_destroy.restype = None
    lib.nam_b200_multi_device_count.argtypes = [C.c_void_p]
    lib.nam_b200_multi_shard.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    lib.nam_b200_multi_reset.argtypes = [C.c_void_p, C.c_double, C.c_int]
    lib.nam_b200_multi_process_f32.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int64]
    lib.nam_b200_measure_fp32_tflops.argtypes = [C.c_int, C.c_int]
    lib.nam_b200_measure_fp32_tflops.restype = C.c_double
    lib.nam_b200_has_tensor_core_kernel.argtypes = []
    lib.nam_b200_has_tensor_core_kernel.restype = C.c_int
    i32p = C.POINTER(C.c_int32)
    lib.nam_b200_stream_state_size.argtypes = [vp]
    lib.nam_b200_stream_state_size.restype = C.c_int64
    lib.nam_b200_reset_streams.argtypes = [vp, i32p, C.c_int, C.c_int]
    lib.nam_b200_copy_streams.argtypes = [vp, i32p, i32p, C.c_int]
    lib.nam_b200_export_streams.argtypes = [vp, i32p, C.c_int, vp, C.c_int64]
    lib.nam_b200_import_streams.argtypes = [vp, i32p, C.c_int, vp, C.c_int64]
    lib.nam_b200_export_streams_device.argtypes = [vp, i32p, C.c_int, vp, C.c_int64, vp]
    lib.nam_b200_import_streams_device.argtypes = [vp, i32p, C.c_int, vp, C.c_int64, vp]
    lib.nam_b200_state_layout_json.argtypes = [C.c_char_p, C.c_char_p, C.c_int64]
    lib.nam_b200_process_streams_f32.argtypes = [vp, i32p, C.c_int, vp, vp, C.c_int, C.c_int64, C.c_int64]
    lib.nam_b200_process_streams_f32_device.argtypes = [vp, i32p, C.c_int, vp, vp, C.c_int, C.c_int64, C.c_int64, vp]
    lib.nam_b200_process_streams_ragged_f32.argtypes = [vp, i32p, C.c_int, i32p, vp, vp, C.c_int64, C.c_int64]
    lib.nam_b200_process_streams_ragged_f32_device.argtypes = [vp, i32p, C.c_int, i32p, vp, vp, C.c_int64, C.c_int64, vp]
    strv = C.POINTER(C.c_char_p)
    lib.nam_b200_create_bank_from_json.argtypes = [strv, C.c_int, C.POINTER(Options), C.POINTER(vp)]
    lib.nam_b200_create_bank_from_files.argtypes = [strv, C.c_int, C.POINTER(Options), C.POINTER(vp)]
    lib.nam_b200_bank_size.argtypes = [vp]
    lib.nam_b200_assign_streams.argtypes = [vp, i32p, C.c_int, i32p]
    lib.nam_b200_stream_models.argtypes = [vp, i32p, C.c_int, i32p]
    lib.nam_b200_bank_model_info.argtypes = [vp, C.c_int, C.POINTER(Info)]
    lib.nam_b200_bank_check_json.argtypes = [strv, C.c_int, C.c_char_p, C.c_int64]
    lib.nam_b200_bank_jit_prepare_json.argtypes = [strv, C.c_int, C.c_int, C.c_char_p, C.c_int64]
    lib.nam_b200_bank_jit_prepare_json.restype = C.c_int
    lib.nam_b200_bank_capacity.argtypes = [vp]
    lib.nam_b200_bank_add_models.argtypes = [vp, strv, C.c_int, i32p]
    lib.nam_b200_bank_replace_model.argtypes = [vp, C.c_int, C.c_char_p]
    lib.nam_b200_resampler_json.argtypes = [C.c_double, C.c_double, C.c_char_p, C.c_int64]
    lib.nam_b200_resampler_json.restype = C.c_int
    for name in ("nam_b200_create_bank_from_json", "nam_b200_create_bank_from_files", "nam_b200_bank_size",
                 "nam_b200_assign_streams", "nam_b200_stream_models", "nam_b200_bank_model_info", "nam_b200_bank_check_json",
                 "nam_b200_bank_capacity", "nam_b200_bank_add_models", "nam_b200_bank_replace_model"):
        getattr(lib, name).restype = C.c_int
    for name in ("nam_b200_reset_streams", "nam_b200_copy_streams", "nam_b200_export_streams", "nam_b200_import_streams",
                 "nam_b200_export_streams_device", "nam_b200_import_streams_device", "nam_b200_state_layout_json",
                 "nam_b200_process_streams_f32", "nam_b200_process_streams_f32_device",
                 "nam_b200_process_streams_ragged_f32", "nam_b200_process_streams_ragged_f32_device"):
        getattr(lib, name).restype = C.c_int
    for name in (
        "nam_b200_create_from_file",
        "nam_b200_create_from_json",
        "nam_b200_get_info",
        "nam_b200_reset",
        "nam_b200_prewarm",
        "nam_b200_process_f32",
        "nam_b200_process_f32_device",
        "nam_b200_process_f64_planar",
        "nam_b200_process_f32_planar",
        "nam_b200_set_fast_tanh",
        "nam_b200_set_reserved_sms",
        "nam_b200_set_slimmable_size",
        "nam_b200_slimmable_breakpoints",
        "nam_b200_synchronize",
    ):
        getattr(lib, name).restype = C.c_int
    _lib = lib
    return lib
