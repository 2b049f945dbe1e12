"""Python mirror of the reference's operator interface for the hot path, on top of the C ABI.

Names and argument meaning follow nam::DSP / nam::get_dsp (reference NAM/dsp.h:70-231,
NAM/get_dsp.h:85-116) so the parity tests read like the reference's own tests:

    model = get_dsp("model.nam", batch=4096)        # nam::get_dsp(path)
    model.Reset(48000.0, 4096)                      # DSP::Reset(sampleRate, maxBufferSize)  (+ prewarm)
    model.process(inp, out, n)                      # DSP::process(NAM_SAMPLE** in, NAM_SAMPLE** out, n), stream 0
    y = model.process_batch(x)                      # the batched reframing: x[batch, n] float32 -> y[batch, n]

There is no CPU path behind this module: every call goes to libnam_b200.so (hand-written sm_90a
kernels) and raises if the library or a CUDA device is missing.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
from typing import Optional

import numpy as np

from . import _capi

# nam_b200_status (include/nam_b200.h)
ERR_INVALID_ARGUMENT, ERR_FILE, ERR_MODEL, ERR_UNSUPPORTED, ERR_CUDA, ERR_STATE = -1, -2, -3, -4, -5, -6


class NamFileValidationError(RuntimeError):
    """nam::NamFileValidationError (NAM/nam_file.h:11-15)."""


class UnsupportedModelError(RuntimeError):
    """Valid .nam, but uses an option the CUDA path does not implement yet."""


class CudaUnavailableError(RuntimeError):
    """No CUDA device / CUDA failure.  The product has no CPU fallback."""


# mirrors nam::activations::Activation::using_fast_tanh (NAM/activations.cpp:16): a process-wide switch
# that must be set BEFORE loading a model (NAM/activations.cpp:168-177).
_using_fast_tanh = False


def enable_fast_tanh() -> None:
    global _using_fast_tanh
    _using_fast_tanh = True


def disable_fast_tanh() -> None:
    global _using_fast_tanh
    _using_fast_tanh = False


def using_fast_tanh() -> bool:
    return _using_fast_tanh


def _raise(rc: int, lib) -> None:
    msg = lib.nam_b200_last_error().decode(errors="replace")
    if rc == ERR_FILE:
        raise NamFileValidationError(msg)
    if rc == ERR_UNSUPPORTED:
        raise UnsupportedModelError(msg)
    if rc == ERR_CUDA:
        raise CudaUnavailableError(msg)
    if rc == ERR_INVALID_ARGUMENT:
        raise ValueError(msg)
    raise RuntimeError(msg)


class DSP:
    """One loaded model carrying `batch` independent streams of device-resident state."""

    def __init__(self, handle: int, lib, batch: int):
        self._h = C.c_void_p(handle)
        self._lib = lib
        self._batch = batch
        self._info = _capi.Info()
        self._refresh_info()

    # ---- lifetime -----------------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.nam_b200_destroy(self._h)
            self._h = C.c_void_p(None)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _refresh_info(self) -> None:
        self._info.struct_size = C.sizeof(_capi.Info)
        rc = self._lib.nam_b200_get_info(self._h, C.byref(self._info))
        if rc != 0:
            _raise(rc, self._lib)

    # ---- nam::DSP accessors (NAM/dsp.h:100-205) -------------------------------------------------
    def GetExpectedSampleRate(self) -> float:
        return self._info.expected_sample_rate

    def NumInputChannels(self) -> int:
        return self._info.in_channels

    def NumOutputChannels(self) -> int:
        return self._info.out_channels

    @property
    def in_channels(self) -> int:
        return self._info.in_channels

    @property
    def out_channels(self) -> int:
        return self._info.out_channels

    def GetPrewarmSamples(self) -> int:
        return self._info.prewarm_samples

    def GetMaxBufferSize(self) -> int:
        self._refresh_info()
        return self._info.max_frames

    def HasLoudness(self) -> bool:
        return bool(self._info.has_loudness)

    def GetLoudness(self) -> float:
        if not self.HasLoudness():
            raise RuntimeError("Asked for loudness of a model that doesn't know how loud it is!")  # dsp.cpp:121-128
        return self._info.loudness

    def HasInputLevel(self) -> bool:
        return bool(self._info.has_input_level)

    def GetInputLevel(self) -> float:
        return self._info.input_level_dbu

    def HasOutputLevel(self) -> bool:
        return bool(self._info.has_output_level)

    def GetOutputLevel(self) -> float:
        return self._info.output_level_dbu

    # ---- extras of the batched reframing --------------------------------------------------------
    @property
    def batch(self) -> int:
        return self._batch

    @property
    def info(self) -> _capi.Info:
        self._refresh_info()
        return self._info

    @property
    def flops_per_frame(self) -> float:
        return self._info.flops_per_frame

    @property
    def state_bytes_per_stream(self) -> int:
        return self._info.state_bytes_per_stream

    @property
    def jit_state(self) -> int:
        """1 = the model-specialised (NVRTC) kernel serves this handle's throughput calls, 0 = not requested,
        -1 = requested but unavailable (jit_note says why)."""
        self._refresh_info()
        return int(self._info.jit_state)

    @property
    def jit_lat_state(self) -> int:
        """The same for the low-latency kernel (few streams, short calls; built by Reset when jit is 1 or 3)."""
        self._refresh_info()
        return int(self._info.jit_lat_state)

    def jit_note(self) -> str:
        buf = C.create_string_buffer(4096)
        self._lib.nam_b200_jit_note(self._h, buf, len(buf))
        return buf.value.decode(errors="replace")

    def launch_count(self) -> int:
        return int(self._lib.nam_b200_launch_count(self._h))

    def last_kernel_ms(self) -> float:
        return float(self._lib.nam_b200_last_kernel_ms(self._h))

    def synchronize(self) -> None:
        rc = self._lib.nam_b200_synchronize(self._h)
        if rc != 0:
            _raise(rc, self._lib)

    # ---- nam::DSP::Reset / prewarm --------------------------------------------------------------
    def Reset(self, sampleRate: float, maxBufferSize: int) -> None:
        rc = self._lib.nam_b200_reset(self._h, float(sampleRate), int(maxBufferSize))
        if rc != 0:
            _raise(rc, self._lib)
        self._refresh_info()

    def prewarm(self) -> None:
        rc = self._lib.nam_b200_prewarm(self._h)
        if rc != 0:
            _raise(rc, self._lib)

    def set_reserved_sms(self, n_sms: int) -> None:
        """Leave n_sms SMs free for concurrent kernels (e.g. an NCCL collective) during the persistent WaveNet kernels."""
        rc = self._lib.nam_b200_set_reserved_sms(self._h, int(n_sms))
        if rc != 0:
            _raise(rc, self._lib)

    def set_fast_tanh(self, enabled: bool) -> None:
        """LSTM reads the switch at run time (NAM/lstm.cpp:48)."""
        self._lib.nam_b200_set_fast_tanh(self._h, int(bool(enabled)))

    # ---- nam::SlimmableModel (NAM/slimmable.h:13-29; ContainerModel, NAM/container.cpp:88-133) ---------
    def SetSlimmableSize(self, val: float) -> None:
        """0.0 = smallest, 1.0 = full size.  Only "SlimmableContainer" files are slimmable."""
        rc = self._lib.nam_b200_set_slimmable_size(self._h, float(val))
        if rc < 0:
            _raise(rc, self._lib)
        self._refresh_info()

    def GetSlimmableSizeBreakpoints(self) -> list:
        n = self._lib.nam_b200_slimmable_breakpoints(self._h, None, 0)
        if n <= 0:
            return []
        buf = (_capi.C.c_double * n)()
        self._lib.nam_b200_slimmable_breakpoints(self._h, buf, n)
        return list(buf)

    # ---- nam::DSP::process ----------------------------------------------------------------------
    def process(self, input, output, num_frames: int) -> None:
        """DSP::process(NAM_SAMPLE** input, NAM_SAMPLE** output, num_frames) for stream 0.

        `input` / `output`: sequences of per-channel 1-D numpy arrays (float64 = NAM_SAMPLE default,
        or float32 = -DNAM_SAMPLE_FLOAT), output written in place.
        """
        n = int(num_frames)
        ins = [np.ascontiguousarray(a) for a in input]
        outs = list(output)
        # the C side reads in_channels pointers and writes out_channels pointers of n frames each: check all of it here
        if len(ins) != self.in_channels or len(outs) != self.out_channels:
            raise ValueError(f"process() needs {self.in_channels} input and {self.out_channels} output channel buffers "
                             f"(got {len(ins)} and {len(outs)})")
        if n < 0 or any(a.ndim != 1 or len(a) < n or a.dtype != ins[0].dtype for a in ins):
            raise ValueError("input buffers must be 1-D, of one dtype, and hold num_frames")
        if ins[0].dtype == np.float64:
            ptr_t, fn = _capi.f64p, self._lib.nam_b200_process_f64_planar
        elif ins[0].dtype == np.float32:
            ptr_t, fn = _capi.f32p, self._lib.nam_b200_process_f32_planar
        else:
            raise TypeError("process() takes float64 (NAM_SAMPLE) or float32 (NAM_SAMPLE_FLOAT) buffers")
        for o in outs:
            if not isinstance(o, np.ndarray) or o.ndim != 1 or o.dtype != ins[0].dtype or not o.flags["C_CONTIGUOUS"] or len(o) < n:
                raise ValueError("output buffers must be contiguous, of the input dtype, and hold num_frames")
        ip = (ptr_t * len(ins))(*[a.ctypes.data_as(ptr_t) for a in ins])
        op = (ptr_t * len(outs))(*[o.ctypes.data_as(ptr_t) for o in outs])
        rc = fn(self._h, ip, op, n)
        if rc != 0:
            _raise(rc, self._lib)

    def process_batch(self, x: np.ndarray, out: Optional[np.ndarray] = None) -> np.ndarray:
        """x: (batch, n) float32 host array, one row per independent stream -> (batch, n) float32.
        Multi-channel models: x (batch, in_channels, n) -> (batch, out_channels, n)."""
        if x.ndim == 3:
            return self._process_batch_multichannel(x, out)
        if x.ndim != 2 or x.dtype != np.float32:
            raise TypeError("process_batch takes a 2-D float32 array [batch, frames]")
        if self.in_channels != 1 or self.out_channels != 1:
            raise TypeError("multi-channel model: process_batch takes [batch, in_channels, frames]")
        if not x.flags["C_CONTIGUOUS"]:
            x = np.ascontiguousarray(x)
        b, n = x.shape
        if out is None:
            out = np.empty_like(x)
        elif (not isinstance(out, np.ndarray) or out.dtype != np.float32 or out.shape != x.shape
              or not out.flags["C_CONTIGUOUS"]):
            raise ValueError("out must be a C-contiguous float32 array of x's shape")  # the C side writes b rows of n floats
        # numpy may report an arbitrary stride for a length-1 axis
        xs = x.strides[0] // 4 if b > 1 else n
        os_ = out.strides[0] // 4 if b > 1 else n
        rc = self._lib.nam_b200_process_f32(self._h, x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), b, n, xs, os_)
        if rc != 0:
            _raise(rc, self._lib)
        return out

    def _process_batch_multichannel(self, x: np.ndarray, out: Optional[np.ndarray]) -> np.ndarray:
        if x.dtype != np.float32 or x.shape[1] != self.in_channels:
            raise TypeError(f"process_batch takes a float32 array [batch, {self.in_channels}, frames]")
        x = np.ascontiguousarray(x)
        b, ci, n = x.shape
        co = self.out_channels
        if out is None:
            out = np.empty((b, co, n), np.float32)
        elif out.shape != (b, co, n) or out.dtype != np.float32 or not out.flags["C_CONTIGUOUS"]:
            raise ValueError(f"out must be a contiguous float32 array [batch, {co}, frames]")
        rc = self._lib.nam_b200_process_f32(self._h, x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), b, n,
                                            ci * n, co * n)
        if rc != 0:
            _raise(rc, self._lib)
        return out

    def process_batch_device(self, in_ptr: int, out_ptr: int, batch: int, n_frames: int, in_stride: int | None = None,
                             out_stride: int | None = None, cuda_stream: int = 0) -> None:
        """Device pointers (e.g. torch.Tensor.data_ptr()), asynchronous on `cuda_stream` (0 = handle's stream)."""
        rc = self._lib.nam_b200_process_f32_device(
            self._h, C.c_void_p(in_ptr), C.c_void_p(out_ptr), int(batch), int(n_frames),
            int(in_stride if in_stride is not None else n_frames), int(out_stride if out_stride is not None else n_frames),
            C.c_void_p(cuda_stream) if cuda_stream else None,
        )
        if rc != 0:
            _raise(rc, self._lib)


def _options(lib, batch: int, device: int, prewarm: Optional[bool], fast_tanh: Optional[bool], ctas_per_sm: int,
             kernel_geometry: int = 0, tile_mode: int = 0, jit: int = 0):
    o = _capi.Options()
    lib.nam_b200_default_options(C.byref(o))
    o.device = int(device)
    o.max_batch = int(batch)
    o.fast_tanh = int(_using_fast_tanh if fast_tanh is None else bool(fast_tanh))
    o.prewarm_on_reset = 1 if prewarm is None else int(bool(prewarm))
    o.ctas_per_sm = int(ctas_per_sm)
    o.kernel_geometry = int(kernel_geometry)
    o.tile_mode = int(tile_mode)
    o.jit = int(jit)
    return o


def get_dsp(config, batch: int = 1, device: int = -1, prewarm: Optional[bool] = None,
            fast_tanh: Optional[bool] = None, ctas_per_sm: int = 0, kernel_geometry: int = 0,
            tile_mode: int = 0, jit: int = 0) -> DSP:
    """nam::get_dsp: `config` is a path to a .nam file, a dict (parsed .nam) or a JSON string.

    batch      number of independent streams the handle carries (the reference: one DSP object each)
    prewarm    DspLoadOptions.prewarm (NAM/get_dsp.h:70-78): None = reference default (Reset prewarms)
    fast_tanh  None = use the process-wide switch (enable_fast_tanh()), like the reference
    kernel_geometry / tile_mode / ctas_per_sm   tuning knobs, see nam_b200_options (include/nam_b200.h)
    jit         model-specialised kernel (NVRTC at load): 0 = default (on for batch >= 256), 1 = required, 2 = off
    """
    import json

    lib = _capi.load()
    o = _options(lib, batch, device, prewarm, fast_tanh, ctas_per_sm, kernel_geometry, tile_mode, jit)
    h = C.c_void_p()
    if isinstance(config, (str, os.PathLike)) and not (isinstance(config, str) and config.lstrip().startswith("{")):
        rc = lib.nam_b200_create_from_file(str(Path(config)).encode(), C.byref(o), C.byref(h))
    else:
        text = config if isinstance(config, str) else json.dumps(config)
        rc = lib.nam_b200_create_from_json(text.encode(), C.byref(o), C.byref(h))
    if rc != 0:
        _raise(rc, lib)
    return DSP(h.value, lib, int(batch))


def jit_prepare(config, fast_tanh: Optional[bool] = None, batch: int = 1) -> dict:
    """Host-only: compile (or fetch from the cache) the model-specialised kernel of a WaveNet .nam (path, dict or JSON
    text).  Needs no GPU: NVRTC cross-compiles for sm_90a.  Returns the library's report as a dict."""
    import json

    lib = _capi.load()
    if isinstance(config, (str, os.PathLike)) and not (isinstance(config, str) and config.lstrip().startswith("{")):
        text = Path(config).read_text()
    else:
        text = config if isinstance(config, str) else json.dumps(config)
    ft = int(_using_fast_tanh if fast_tanh is None else bool(fast_tanh))
    buf = C.create_string_buffer(2048)
    rc = lib.nam_b200_jit_prepare_json_for_batch(text.encode(), ft, int(batch), buf, len(buf))
    if rc != 0:
        _raise(rc, lib)
    return json.loads(buf.value.decode())


def inspect(config, fast_tanh: Optional[bool] = None) -> dict:
    """Host-only: parse/validate a .nam (path, dict or JSON text) with the product's C++ loader and report
    what the CUDA path would do with it.  Needs no GPU."""
    import json

    lib = _capi.load()
    buf = C.create_string_buffer(2048)
    ft = int(_using_fast_tanh if fast_tanh is None else bool(fast_tanh))
    if isinstance(config, (str, os.PathLike)) and not (isinstance(config, str) and config.lstrip().startswith("{")):
        rc = lib.nam_b200_inspect_file(str(Path(config)).encode(), ft, buf, len(buf))
    else:
        text = config if isinstance(config, str) else json.dumps(config)
        rc = lib.nam_b200_inspect_json(text.encode(), ft, buf, len(buf))
    if rc != 0:
        _raise(rc, lib)
    return json.loads(buf.value.decode())


def submodels(config) -> list:
    """Host-only: the sub-models of a slimmable document as [(max_value, .nam dict), ...] -- the entries of a
    SlimmableContainer file, or the sliced plain WaveNets a "slimmable" WaveNet (NAM/wavenet/slimmable.cpp) stands for.
    [] for a model that is not slimmable.  Needs no GPU."""
    import json

    lib = _capi.load()
    text = (Path(config).read_text() if isinstance(config, os.PathLike) or (isinstance(config, str) and not config.lstrip().startswith("{"))
            else (config if isinstance(config, str) else json.dumps(config))).encode()
    n = lib.nam_b200_submodel_json(text, -1, None, None, 0)
    if n < 0:
        _raise(int(n), lib)
    out = []
    for i in range(int(n)):
        mv = C.c_double()
        size = lib.nam_b200_submodel_json(text, i, C.byref(mv), None, 0)
        if size < 0:
            _raise(int(size), lib)
        buf = C.create_string_buffer(int(size) + 1)
        lib.nam_b200_submodel_json(text, i, C.byref(mv), buf, len(buf))
        out.append((mv.value, json.loads(buf.value.decode())))
    return out


def has_tensor_core_kernel() -> bool:
    """Does libnam_b200.so have a tensor-core WaveNet kernel (kernel_geometry=3)?  Never on sm_90a."""
    return bool(_capi.load().nam_b200_has_tensor_core_kernel())


def measure_fp32_tflops(device: int = -1, packed: bool = True) -> float:
    """Measured FP32 FMA throughput of the device (the compute roofline of the fused kernel)."""
    return float(_capi.load().nam_b200_measure_fp32_tflops(int(device), int(packed)))
