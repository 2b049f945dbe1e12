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

    @property
    def resample_ratio(self) -> tuple:
        """(L, M): the conversion of the last Reset, model rate / host rate = L / M; (1, 1) when none."""
        self._refresh_info()
        return int(self._info.resample_up), int(self._info.resample_down)

    @property
    def resample_latency(self) -> int:
        """Group delay of the conversion in host frames, rounded (resampler()['latency_frames'] exactly); 0 when none."""
        self._refresh_info()
        return int(self._info.resample_latency_frames)

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

    def process_streams(self, streams, x: np.ndarray, out: Optional[np.ndarray] = None, n_frames=None) -> np.ndarray:
        """Run only the listed streams (distinct, any order): row i of x belongs to streams[i], and each stream continues
        from its own history, however many calls it sat out; unlisted streams are untouched.  x: (n, frames) float32, or
        (n, in_channels, frames) for a multi-channel model -> out of the same layout with out_channels.

        n_frames (a sequence, one count per row): a ragged call -- row i runs only its first n_frames[i] frames, frames is
        max(n_frames), the rest of the row is padding that is never read and comes back as zeros; each stream advances
        by its own count (0: the stream is left exactly as it was)."""
        s = self._streams(streams)
        x = np.asarray(x)
        if x.ndim == 3:
            if x.dtype != np.float32 or x.shape[1] != self.in_channels:
                raise TypeError(f"process_streams takes a float32 array [n, {self.in_channels}, frames]")
            n_rows, _, n = x.shape
            shape = (n_rows, self.out_channels, n)
        else:
            if x.ndim != 2 or x.dtype != np.float32:
                raise TypeError("process_streams takes a 2-D float32 array [n, frames]")
            if self.in_channels != 1 or self.out_channels != 1:
                raise TypeError("multi-channel model: process_streams takes [n, in_channels, frames]")
            n_rows, n = x.shape
            shape = (n_rows, n)
        if n_rows != len(s):
            raise ValueError(f"x has {n_rows} rows for {len(s)} streams")
        x = np.ascontiguousarray(x)
        if out is None:
            out = np.empty(shape, np.float32)
        elif (not isinstance(out, np.ndarray) or out.dtype != np.float32 or out.shape != shape
              or not out.flags["C_CONTIGUOUS"]):
            raise ValueError(f"out must be a C-contiguous float32 array of shape {shape}")
        if n_frames is None:
            self._check(self._lib.nam_b200_process_streams_f32(self._h, self._i32p(s), len(s), x.ctypes.data_as(C.c_void_p),
                                                               out.ctypes.data_as(C.c_void_p), n, self.in_channels * n,
                                                               self.out_channels * n))
            return out
        counts = self._counts(n_frames, len(s))
        if len(counts) and int(counts.max()) != n:
            raise ValueError(f"x has {n} frames per row; a ragged call takes max(n_frames) = {int(counts.max())}")
        self._check(self._lib.nam_b200_process_streams_ragged_f32(
            self._h, self._i32p(s), len(s), self._i32p(counts), x.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p),
            self.in_channels * n, self.out_channels * n))
        return out

    def process_streams_device(self, streams, in_ptr: int, out_ptr: int, n_frames, in_stride: int | None = None,
                               out_stride: int | None = None, cuda_stream: int = 0) -> None:
        """process_streams on device buffers (e.g. torch.Tensor.data_ptr()), asynchronous on `cuda_stream` (0 = the
        handle's stream).  Strides in floats between rows, default channels x n_frames.  n_frames: an int, or a sequence
        of one count per row for a ragged call (rows laid out at a pitch of max(n_frames), padding neither read nor
        written)."""
        s = self._streams(streams)
        st = C.c_void_p(cuda_stream) if cuda_stream else None
        if isinstance(n_frames, (int, np.integer)):
            self._check(self._lib.nam_b200_process_streams_f32_device(
                self._h, self._i32p(s), len(s), C.c_void_p(in_ptr), C.c_void_p(out_ptr), int(n_frames),
                int(in_stride if in_stride is not None else self.in_channels * n_frames),
                int(out_stride if out_stride is not None else self.out_channels * n_frames), st))
            return
        counts = self._counts(n_frames, len(s))
        n_max = int(counts.max()) if len(counts) else 0
        self._check(self._lib.nam_b200_process_streams_ragged_f32_device(
            self._h, self._i32p(s), len(s), self._i32p(counts), C.c_void_p(in_ptr), C.c_void_p(out_ptr),
            int(in_stride if in_stride is not None else self.in_channels * n_max),
            int(out_stride if out_stride is not None else self.out_channels * n_max), st))

    @staticmethod
    def _counts(n_frames, n: int) -> np.ndarray:
        """Per-row frame counts of a ragged call -> int32 array (range checks are the library's)."""
        counts = np.ascontiguousarray(np.asarray(n_frames, dtype=np.int64).reshape(-1))
        if len(counts) != n:
            raise ValueError(f"n_frames has {len(counts)} entries for {n} streams")
        if len(counts) and (counts.min() < np.iinfo(np.int32).min or counts.max() > np.iinfo(np.int32).max):
            raise ValueError("n_frames entries must fit in int32")
        return counts.astype(np.int32)

    # ---- per-stream state (include/nam_b200.h: records, per-stream clocks) ------------------------------------------
    @property
    def state_record_bytes(self) -> int:
        """Bytes of one stream's state record (64-byte header + float32 payload)."""
        n = int(self._lib.nam_b200_stream_state_size(self._h))
        if n < 0:
            _raise(n, self._lib)
        return n

    @staticmethod
    def _streams(streams) -> np.ndarray:
        return np.ascontiguousarray(np.atleast_1d(np.asarray(streams)), dtype=np.int32)

    @staticmethod
    def _i32p(a: np.ndarray):
        return a.ctypes.data_as(C.POINTER(C.c_int32))

    def _check(self, rc: int) -> None:
        if rc != 0:
            _raise(rc, self._lib)

    def reset_streams(self, streams, fresh: bool = False) -> None:
        """DSP::Reset for the listed streams only (the others are untouched).  LSTM: fresh=False keeps h, c and prewarms
        on top of them (what Reset does); fresh=True starts from the trained initial state like a new handle."""
        s = self._streams(streams)
        self._check(self._lib.nam_b200_reset_streams(self._h, self._i32p(s), len(s), int(bool(fresh))))

    def copy_streams(self, src, dst) -> None:
        """dst[i] takes src[i]'s state; the sources are all read first, so a swap works."""
        s, d = self._streams(src), self._streams(dst)
        if len(s) != len(d):
            raise ValueError("src and dst must list the same number of streams")
        self._check(self._lib.nam_b200_copy_streams(self._h, self._i32p(s), self._i32p(d), len(s)))

    def export_streams(self, streams) -> np.ndarray:
        """The listed streams' state records -> uint8 array (n, state_record_bytes)."""
        s = self._streams(streams)
        rb = self.state_record_bytes
        out = np.zeros((len(s), rb), np.uint8)
        self._check(self._lib.nam_b200_export_streams(self._h, self._i32p(s), len(s), out.ctypes.data_as(C.c_void_p), rb))
        return out

    def import_streams(self, streams, records: np.ndarray) -> None:
        """Records (one row each, as export_streams returns them) -> the listed streams."""
        s = self._streams(streams)
        r = np.asarray(records)
        if r.ndim == 1:
            r = r[None, :]
        if r.dtype != np.uint8 or r.ndim != 2 or r.shape[0] != len(s):
            raise ValueError("records must be a uint8 array with one row per stream")
        r = np.ascontiguousarray(r)
        self._check(self._lib.nam_b200_import_streams(self._h, self._i32p(s), len(s), r.ctypes.data_as(C.c_void_p), r.shape[1]))

    def export_streams_device(self, streams, dst_ptr: int, record_stride: int | None = None, cuda_stream: int = 0) -> None:
        """Records into device memory at dst_ptr (e.g. torch.Tensor.data_ptr()), asynchronous on `cuda_stream`."""
        s = self._streams(streams)
        stride = int(record_stride if record_stride is not None else self.state_record_bytes)
        self._check(self._lib.nam_b200_export_streams_device(self._h, self._i32p(s), len(s), C.c_void_p(dst_ptr), stride,
                                                             C.c_void_p(cuda_stream) if cuda_stream else None))

    def import_streams_device(self, streams, src_ptr: int, record_stride: int | None = None, cuda_stream: int = 0) -> None:
        """Records from device memory -> the listed streams; the headers are checked on the host before any launch."""
        s = self._streams(streams)
        stride = int(record_stride if record_stride is not None else self.state_record_bytes)
        self._check(self._lib.nam_b200_import_streams_device(self._h, self._i32p(s), len(s), C.c_void_p(src_ptr), stride,
                                                             C.c_void_p(cuda_stream) if cuda_stream else None))

    # ---- model banks (nam_b200_create_bank_*) --------------------------------------------------------------------------
    @property
    def bank_size(self) -> int:
        """K of a bank (get_dsp_bank); 1 for an ordinary handle."""
        n = int(self._lib.nam_b200_bank_size(self._h))
        if n < 0:
            _raise(n, self._lib)
        return n

    def assign_streams(self, streams, models) -> None:
        """Bind streams[i] to model models[i] and give it that model's freshly reset state; other streams are untouched.
        On an ordinary handle, models all 0 is reset_streams (for an LSTM: fresh=False, which keeps the running state); on
        a bank it is reset_streams(fresh=True) on an ordinary handle of the new model."""
        s = self._streams(streams)
        k = np.ascontiguousarray(np.broadcast_to(np.asarray(models, dtype=np.int32), s.shape), dtype=np.int32)
        self._check(self._lib.nam_b200_assign_streams(self._h, self._i32p(s), len(s), self._i32p(k)))

    def stream_models(self, streams) -> np.ndarray:
        """The model each listed stream is bound to (int32 array)."""
        s = self._streams(streams)
        out = np.zeros(len(s), np.int32)
        self._check(self._lib.nam_b200_stream_models(self._h, self._i32p(s), len(s), self._i32p(out)))
        return out

    def model_info(self, k: int) -> _capi.Info:
        """get_info with model k's loudness, levels, expected sample rate and weight count."""
        info = _capi.Info()
        info.struct_size = C.sizeof(_capi.Info)
        self._check(self._lib.nam_b200_bank_model_info(self._h, int(k), C.byref(info)))
        return info

    @property
    def bank_capacity(self) -> int:
        """Models this bank can hold (get_dsp_bank's capacity; K when it was created with 0); 1 for an ordinary handle."""
        n = int(self._lib.nam_b200_bank_capacity(self._h))
        if n < 0:
            _raise(n, self._lib)
        return n

    def add_models(self, configs) -> list:
        """Add documents (paths, dicts or JSON texts) of the bank's shape as models K, K+1, ...; returns their indices.
        All or nothing: a document that could not join the bank at creation, or more documents than the capacity leaves
        room for, raise and leave the bank unchanged.  After a reset the new models' fresh states are prepared at once;
        no stream's state changes."""
        arr, keep = _text_array(_documents(configs))
        first = C.c_int32(0)
        self._check(self._lib.nam_b200_bank_add_models(self._h, arr, len(keep), C.byref(first)))
        return list(range(first.value, first.value + len(keep)))

    def replace_model(self, k: int, config) -> None:
        """Model k takes another document of the bank's shape (path, dict or JSON text).  Refused while a stream is bound
        to k (move those streams with assign_streams first); waits for every earlier call of the bank to finish with the
        old weights."""
        self._check(self._lib.nam_b200_bank_replace_model(self._h, int(k), _documents([config])[0].encode()))


def _options(lib, batch: int, device: int, prewarm: Optional[bool], fast_tanh: Optional[bool], ctas_per_sm: int,
             kernel_geometry: int = 0, tile_mode: int = 0, jit: int = 0, capacity: int = 0, resample: bool = False):
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
    o.bank_capacity = int(capacity)
    o.resample = int(bool(resample))
    return o


def get_dsp(config, batch: int = 1, device: int = -1, prewarm: Optional[bool] = None,
            fast_tanh: Optional[bool] = None, ctas_per_sm: int = 0, kernel_geometry: int = 0,
            tile_mode: int = 0, jit: int = 0, resample: bool = False) -> DSP:
    """nam::get_dsp: `config` is a path to a .nam file, a dict (parsed .nam) or a JSON string.

    batch      number of independent streams the handle carries (the reference: one DSP object each)
    prewarm    DspLoadOptions.prewarm (NAM/get_dsp.h:70-78): None = reference default (Reset prewarms)
    fast_tanh  None = use the process-wide switch (enable_fast_tanh()), like the reference
    kernel_geometry / tile_mode / ctas_per_sm   tuning knobs, see nam_b200_options (include/nam_b200.h)
    jit         model-specialised kernel (NVRTC at load): 0 = default (on for batch >= 256), 1 = required, 2 = off
    resample    True = Reset(sampleRate) at a rate other than the model's converts every stream to the model's rate and
                back on the device (resampler(); DSP.resample_ratio, DSP.resample_latency); False = the reference's
                behaviour: the rate is recorded and ignored
    """
    import json

    lib = _capi.load()
    o = _options(lib, batch, device, prewarm, fast_tanh, ctas_per_sm, kernel_geometry, tile_mode, jit, resample=resample)
    h = C.c_void_p()
    if isinstance(config, (str, os.PathLike)) and not (isinstance(config, str) and config.lstrip().startswith("{")):
        rc = lib.nam_b200_create_from_file(str(Path(config)).encode(), C.byref(o), C.byref(h))
    else:
        text = config if isinstance(config, str) else json.dumps(config)
        rc = lib.nam_b200_create_from_json(text.encode(), C.byref(o), C.byref(h))
    if rc != 0:
        _raise(rc, lib)
    return DSP(h.value, lib, int(batch))


def _documents(configs) -> list:
    """.nam paths, dicts or JSON texts -> JSON texts"""
    import json

    out = []
    for c in configs:
        if isinstance(c, (str, os.PathLike)) and not (isinstance(c, str) and c.lstrip().startswith("{")):
            out.append(Path(c).read_text())
        else:
            out.append(c if isinstance(c, str) else json.dumps(c))
    return out


def _text_array(texts: list):
    enc = [t.encode() for t in texts]
    return (C.c_char_p * max(len(enc), 1))(*enc), enc


def get_dsp_bank(configs, batch: int = 1, device: int = -1, prewarm: Optional[bool] = None,
                 fast_tanh: Optional[bool] = None, ctas_per_sm: int = 0, kernel_geometry: int = 0,
                 tile_mode: int = 0, jit: int = 0, capacity: int = 0, resample: bool = False) -> DSP:
    """A model bank: one handle of `batch` streams over the K documents in `configs` (paths, dicts or JSON texts), which
    must share one shape (bank_check): WaveNets of the fused kernel family, WaveNets of the general kernel (A2-style,
    condition_dsp, multi-channel), ConvNets, or LSTMs.  Every stream starts bound to model
    0; DSP.assign_streams rebinds.  Each stream behaves as the same stream of an ordinary jit=2 handle of its model: an LSTM
    bank's Reset keeps each stream's running state and prewarms it with its own model, reset_streams(fresh=False) does
    the same for the listed streams, and fresh=True gives them their model's h0 / c0 plus the prewarm.  The options are
    get_dsp's.  jit: a general-WaveNet bank takes it as an ordinary handle does, for the general kernel compiled for the
    bank's shape (bank_jit_prepare; 0 default, 1 required, 2 off, 3 preferred); fused and LSTM banks refuse jit = 1 and
    run the precompiled kernels under 0 / 3; a ConvNet bank takes it as an ordinary ConvNet handle.  kernel_geometry = 4
    is refused for fused-family and LSTM banks; on a general bank it selects the precompiled general kernel, and a
    ConvNet bank ignores it.  capacity: the models the bank can hold (0 = len(configs)); room for DSP.add_models is
    reserved at creation.  A bank of one document and capacity 0 or 1 is get_dsp.  resample: as get_dsp's; the bank's
    models share one expected rate, hence one conversion."""
    lib = _capi.load()
    o = _options(lib, batch, device, prewarm, fast_tanh, ctas_per_sm, kernel_geometry, tile_mode, jit, capacity, resample)
    arr, _keep = _text_array(_documents(configs))
    h = C.c_void_p()
    rc = lib.nam_b200_create_bank_from_json(arr, len(_keep), C.byref(o), C.byref(h))
    if rc != 0:
        _raise(rc, lib)
    return DSP(h.value, lib, int(batch))


def bank_check(configs) -> dict:
    """Host-only: can these documents share a bank?  Model 0 chooses the family (fused-kernel WaveNets, general-kernel
    WaveNets, ConvNets or LSTMs); the others must match it in everything but their weights -- for general WaveNets: every
    array, layer, FiLM, head and condition_dsp field, hence the general kernel's descriptors (both output scales and a
    nested condition_dsp's weights and metadata are per model); for ConvNets: channels, dilations, BatchNorm presence and
    activation; for LSTMs: sample rate, in/out channels, num_layers, input_size, hidden_size; always the sample rate and
    the config object.  Fused and general WaveNets do not mix (reason "model k: kernel: ...").  {ok, n_models, reason (first offending model and field), fingerprints
    (each model's state record fingerprint)}.  Needs no GPU."""
    import json

    lib = _capi.load()
    arr, keep = _text_array(_documents(configs))
    buf = C.create_string_buffer(1 << 16)
    rc = lib.nam_b200_bank_check_json(arr, len(keep), buf, len(buf))
    if rc != 0:
        _raise(rc, lib)
    return json.loads(buf.value.decode())


def bank_jit_prepare(configs, fast_tanh: Optional[bool] = None) -> dict:
    """Host-only: compile (or find in the cache) the general kernel compiled for the shape of a bank of general-kernel
    WaveNets (the kernel get_dsp_bank runs for them under jit 0 / 1 / 3).  The cache key holds no weight: every bank of one
    shape shares the cubin.  {ok, from_cache, compile_seconds, cubin_bytes, threads, smem_bytes, why_not}.  Documents that
    cannot share a bank, and banks of other families, raise as get_dsp_bank would.  Needs no GPU."""
    import json

    lib = _capi.load()
    arr, keep = _text_array(_documents(configs))
    ft = int(_using_fast_tanh if fast_tanh is None else bool(fast_tanh))
    buf = C.create_string_buffer(1 << 16)
    rc = lib.nam_b200_bank_jit_prepare_json(arr, len(keep), ft, buf, len(buf))
    if rc != 0:
        _raise(rc, lib)
    return json.loads(buf.value.decode())


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


def resampler(host_rate: float, model_rate: float) -> dict:
    """Host-only: the sample-rate conversion between these rates (get_dsp(resample=True)): L, M (model / host = L / M),
    n_taps, taps_per_output_up / _down, latency_frames (host frames) and the float32 taps g_up, g_dn as numpy arrays.
    Pairs Reset would refuse raise ValueError naming both rates.  Needs no GPU."""
    import json

    lib = _capi.load()
    buf = C.create_string_buffer(1 << 20)
    rc = lib.nam_b200_resampler_json(float(host_rate), float(model_rate), buf, len(buf))
    if rc != 0:
        _raise(rc, lib)
    d = json.loads(buf.value.decode())
    d["g_up"] = np.asarray(d["g_up"], dtype=np.float32)
    d["g_dn"] = np.asarray(d["g_dn"], dtype=np.float32)
    return d


def state_layout(config) -> dict:
    """Host-only: the per-stream state record of a .nam (path, dict or JSON text): architecture, header_bytes,
    payload_floats, record_bytes, fingerprint and segments [{name, channels, columns, offset}].  Needs no GPU."""
    import json

    lib = _capi.load()
    text = (Path(config).read_text() if isinstance(config, os.PathLike) or (isinstance(config, str) and not config.lstrip().startswith("{"))
            else (config if isinstance(config, str) else json.dumps(config))).encode()
    buf = C.create_string_buffer(1 << 20)
    rc = lib.nam_b200_state_layout_json(text, buf, len(buf))
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
