/*
 * nam_b200.h -- C ABI of libnam_b200.so: NeuralAmpModelerCore's inference hot path on H100 (sm_90a).
 *
 * The reference has no FFI of its own (it is a C++ static library); these entry points are what
 * a binding of its public surface for this path needs, one for one:
 *
 *   nam_b200_create_from_file   <->  nam::get_dsp(std::filesystem::path, DspLoadOptions)   NAM/get_dsp.h:85-90
 *   nam_b200_create_from_json   <->  nam::get_dsp(const nlohmann::json&, ...)              NAM/get_dsp.h:108-116
 *   nam_b200_reset              <->  nam::DSP::Reset(sampleRate, maxBufferSize) + prewarm  NAM/dsp.h:165, NAM/dsp.cpp:67-101,130-140
 *   nam_b200_process_f64_planar <->  nam::DSP::process(NAM_SAMPLE**, NAM_SAMPLE**, int)    NAM/dsp.h:97 (NAM_SAMPLE = double)
 *   nam_b200_process_f32_planar <->  same with -DNAM_SAMPLE_FLOAT                          NAM/dsp.h:18-22
 *   nam_b200_process_f32        <->  the batched reframing: `batch` independent streams per call
 *                                    (each stream == one nam::DSP instance of the reference)
 *   nam_b200_get_info           <->  NumInputChannels/NumOutputChannels/GetExpectedSampleRate/
 *                                    GetPrewarmSamples/Has*,Get* level & loudness          NAM/dsp.h:100-231
 *   nam_b200_set_fast_tanh      <->  nam::activations::Activation::enable/disable_fast_tanh NAM/activations.h:163-164
 *   nam_b200_set_slimmable_size <->  nam::SlimmableModel::SetSlimmableSize (ContainerModel)     NAM/slimmable.h:17, NAM/container.cpp:99-122
 *   nam_b200_slimmable_breakpoints <-> GetSlimmableSizeBreakpoints                              NAM/container.cpp:124-133
 *   nam_b200_last_error         <->  the what() of the exception the reference would throw
 *   nam_b200_destroy            <->  ~unique_ptr<nam::DSP>
 *
 * Conventions: every function returns 0 on success or a negative nam_b200_status; nothing
 * throws across this boundary; pointers are plain host pointers unless the name says _device.
 * A handle owns device weights, per-stream state and staging buffers; the caller owns audio
 * buffers.  process_* calls on one handle are not re-entrant (same as nam::DSP::process).
 * There is NO CPU fallback: if no CUDA device is usable, create fails with NAM_B200_ERR_CUDA.
 */
#ifndef NAM_B200_H
#define NAM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NAM_B200_ABI_VERSION 1

typedef struct nam_b200_model nam_b200_model;

typedef enum nam_b200_status
{
  NAM_B200_OK = 0,
  NAM_B200_ERR_INVALID_ARGUMENT = -1,
  NAM_B200_ERR_FILE = -2, /* nam::NamFileValidationError */
  NAM_B200_ERR_MODEL = -3, /* std::runtime_error / std::invalid_argument while parsing or building */
  NAM_B200_ERR_UNSUPPORTED = -4, /* valid .nam, but an option the CUDA path does not implement yet */
  NAM_B200_ERR_CUDA = -5, /* CUDA runtime failure (message carries cudaGetErrorString) */
  NAM_B200_ERR_STATE = -6 /* call sequence error, e.g. process before reset */
} nam_b200_status;

typedef struct nam_b200_options
{
  int32_t struct_size; /* sizeof(nam_b200_options), for forward compatibility */
  int32_t device; /* CUDA device ordinal, -1 = current device */
  int32_t max_batch; /* number of independent streams this handle carries state for (>= 1) */
  int32_t fast_tanh; /* 1 = Activation::enable_fast_tanh() was called before loading (benchmodel default) */
  int32_t prewarm_on_reset; /* 1 (reference default) = reset() prewarms; 0 = SetPrewarmOnReset(false) */
  int32_t ctas_per_sm; /* 0 = library default; tuning knob for the persistent WaveNet kernel */
  int32_t kernel_geometry; /* WaveNet kernel: 0 = library default; 1 = FP32 FFMA kernel, 128-thread CTAs (tile 256);
                              2 = FP32 FFMA kernel, 256-thread CTAs (tile 512); 3 = tensor-core kernel (none in
                              this library: refused); 4 = the general kernel (all WaveNet options, one CTA per stream,
                              thread per frame) that otherwise serves only models outside the fused families */
  int32_t tile_mode; /* few streams x long calls (batch x tiles <= resident CTAs): 0 = library default: lock-step
                        tile-parallel mode (every (stream, tile) its own CTA, all tiles advancing layer by layer; a
                        history buffer of up to ~150 MB is allocated by reset(); tiles of 128 frames while every CTA has
                        an SM to itself, else 256 frames, 128 threads x 2 frames, or 512 frames, 256 x 2, when those do
                        not all fit -- kernel_geometry 1 / 2 pins one of the last two); 1 = wavefront
                        tile-parallel mode (no buffer, tile c one layer behind tile c-1); 2 = never: one CTA walks a
                        stream's tiles in turn.  Tile-parallel launches need their CTAs co-resident: do not run
                        other kernels on the same GPU concurrently with such a call */
  int32_t jit; /* model-specialised WaveNet kernel (the model compiled to SASS by NVRTC at load time, weights as FFMA
                  immediates; cubins cached under $NAM_B200_JIT_CACHE or <library dir>/jit_cache): 0 = library default
                  (on for handles with max_batch >= 256; $NAM_B200_JIT=0/1 overrides), 1 = required (create fails
                  with the reason if NVRTC or the model's shape rules it out), 2 = off, 3 = preferred (like 1, but a
                  handle that cannot have it keeps the precompiled kernels silently; also asks reset() for the
                  low-latency kernel on handles with few streams and maxBufferSize <= 128 -- the C++ shim's default).  Only calls that take the
                  persistent one-CTA-per-stream path use it; every other mode runs the precompiled kernels on the
                  same state */
  int32_t reserved[5];
} nam_b200_options;

typedef struct nam_b200_info
{
  int32_t struct_size;
  int32_t architecture; /* 1 WaveNet, 2 LSTM, 3 Linear, 5 ConvNet (4: a SlimmableContainer reports its active sub-model) */
  int32_t in_channels, out_channels;
  int32_t prewarm_samples; /* DSP::GetPrewarmSamples() */
  int32_t max_batch, max_frames; /* max_frames = maxBufferSize of the last reset (0 before) */
  int32_t has_loudness, has_input_level, has_output_level;
  double expected_sample_rate; /* -1 when unknown */
  double loudness, input_level_dbu, output_level_dbu;
  int64_t n_weights;
  int64_t state_bytes_per_stream; /* device bytes of per-stream history */
  double flops_per_frame; /* algorithmic FLOPs (2 x MACs) per frame per stream */
  int32_t kernel_variant; /* which CUDA specialisation serves this model (diagnostic) */
  int32_t jit_state; /* model-specialised kernel: 1 = active, 0 = not requested, -1 = requested but unavailable */
  int32_t jit_lat_state; /* the same for the low-latency kernel (few streams, calls of <= 128 frames; built by reset) */
  int32_t reserved[5];
} nam_b200_info;

/* Fill with defaults: device -1, max_batch 1, fast_tanh 0, prewarm_on_reset 1. */
void nam_b200_default_options(nam_b200_options* opts);

int nam_b200_abi_version(void);

int nam_b200_create_from_file(const char* nam_path, const nam_b200_options* opts, nam_b200_model** out);
int nam_b200_create_from_json(const char* nam_json_text, const nam_b200_options* opts, nam_b200_model** out);
void nam_b200_destroy(nam_b200_model* m);

int nam_b200_get_info(const nam_b200_model* m, nam_b200_info* info);

/* DSP::Reset: (re)allocate for calls of up to max_frames frames, zero every stream's history, then
 * (unless prewarm_on_reset == 0) prewarm exactly like DSP::prewarm(): zeros in max_frames-sized blocks
 * until >= prewarm_samples were fed.  All max_batch streams end up in the identical prewarmed state. */
int nam_b200_reset(nam_b200_model* m, double sample_rate, int max_frames);

/* DSP::prewarm() on its own (after a reset with prewarm_on_reset == 0). */
int nam_b200_prewarm(nam_b200_model* m);

/* Batched throughput entry: `batch` (<= max_batch) streams, stream b reads
 * in[b*in_stride .. +n_frames) and writes out[b*out_stride .. +n_frames); n_frames <= max_frames.
 * Multi-channel models (in_channels / out_channels of nam_b200_info != 1; WaveNet: NAM/wavenet/model.cpp:809-820,
 * 888-909, LSTM: NAM/lstm.cpp:103-125): a stream's row holds its channel planes back to back, channel c of stream b
 * at in[b*in_stride + c*n_frames .. +n_frames) (out likewise), strides >= channels * n_frames.
 * Host pointers; copies ride the handle's stream; returns after the result is in `out`. */
int nam_b200_process_f32(nam_b200_model* m, const float* in, float* out, int batch, int n_frames, int64_t in_stride,
                         int64_t out_stride);

/* Same, device pointers, asynchronous on `cuda_stream` (a cudaStream_t, may be NULL = handle's stream).
 * No copies, no synchronisation. */
int nam_b200_process_f32_device(nam_b200_model* m, const float* in_device, float* out_device, int batch, int n_frames,
                                int64_t in_stride, int64_t out_stride, void* cuda_stream);

/* Host-buffer contract of nam_b200_process_f32: any host memory is accepted; with PAGE-LOCKED buffers (cudaMallocHost,
 * cudaHostRegister, or nam_b200_pin_host_buffer below) the call pipelines host->device copy, kernel and device->host copy
 * of successive chunks of streams, with pageable buffers the driver stages the copies and that overlap is lost (same
 * results, ~15-20 % slower end to end).  These helpers let a host without the CUDA runtime pin its buffers once. */
int nam_b200_pin_host_buffer(void* ptr, int64_t bytes);
int nam_b200_unpin_host_buffer(void* ptr);
int nam_b200_host_buffer_is_pinned(const void* ptr); /* 1 pinned / device-accessible, 0 pageable, < 0 error */

/* Several GPUs behind one handle (BASELINE.json config 5: the batch shards across GPUs, no collective on the data path:
 * the streams are independent).  `opts->max_batch` = total streams, dealt out in contiguous blocks
 * [max_batch * i / n, max_batch * (i + 1) / n) to devices[i]; `opts->device` is ignored.  process() runs one worker
 * thread per GPU and returns when every shard's results are in `out`; errors name the device. */
typedef struct nam_b200_multi nam_b200_multi;
int nam_b200_multi_create_from_file(const char* nam_path, const nam_b200_options* opts, const int32_t* devices, int n_devices,
                                    nam_b200_multi** out);
int nam_b200_multi_create_from_json(const char* nam_json_text, const nam_b200_options* opts, const int32_t* devices,
                                    int n_devices, nam_b200_multi** out);
void nam_b200_multi_destroy(nam_b200_multi* mm);
int nam_b200_multi_device_count(const nam_b200_multi* mm);
int nam_b200_multi_shard(const nam_b200_multi* mm, int part, int32_t* device, int32_t* first_stream, int32_t* n_streams);
int nam_b200_multi_reset(nam_b200_multi* mm, double sample_rate, int max_frames);
int nam_b200_multi_process_f32(nam_b200_multi* mm, const float* in, float* out, int batch, int n_frames, int64_t in_stride,
                               int64_t out_stride);

/* nam::DSP::process for stream 0 of the handle: planar input[channel][frame], in_channels input arrays and
 * out_channels output arrays like the reference's NAM_SAMPLE** (NAM/dsp.h:97). */
int nam_b200_process_f64_planar(nam_b200_model* m, const double* const* input, double* const* output, int n_frames);
int nam_b200_process_f32_planar(nam_b200_model* m, const float* const* input, float* const* output, int n_frames);

/* 1 when the library has a tensor-core WaveNet kernel (options.kernel_geometry = 3), else 0: creating a handle with
 * kernel_geometry = 3 then fails with NAM_B200_ERR_UNSUPPORTED.  The sm_90a library has none (0). */
int nam_b200_has_tensor_core_kernel(void);

/* The persistent WaveNet throughput kernels occupy every SM for a whole call, so a concurrent kernel on another stream (an NCCL
 * collective gathering the previous call's outputs, say) only starts when they drain.  Leaving `n_sms` SMs free (0 = none,
 * the default) lets such work overlap the call.  The price is
 * quantised: the streams are walked in rounds of (CTAs per SM) x (SMs left), so check that the batch does not need one more
 * round (4096 streams, 2 CTAs per SM: 16 rounds on 128 to 132 SMs, 17 on 127 or fewer). */
int nam_b200_set_reserved_sms(nam_b200_model* m, int n_sms);

/* LSTM reads the fast-tanh switch at run time (NAM/lstm.cpp:48); WaveNet captured it at load. */
int nam_b200_set_fast_tanh(nam_b200_model* m, int enabled);

/* nam::SlimmableModel (NAM/slimmable.h:13-29) for "SlimmableContainer" files (NAM/container.cpp:88-133): pick the
 * sub-model whose max_value is the first one above `value` (the last one if none is); a newly selected sub-model is
 * reset + prewarmed with the settings of the container's last reset before it takes over.  Every other call on the
 * handle (process, info, prewarm ...) is served by the active sub-model.  Returns 1 if another sub-model became
 * active, 0 if the active one already matched; not slimmable -> NAM_B200_ERR_UNSUPPORTED. */
int nam_b200_set_slimmable_size(nam_b200_model* m, double value);
/* GetSlimmableSizeBreakpoints(): writes up to `capacity` thresholds, returns how many there are (0 = not slimmable). */
int nam_b200_slimmable_breakpoints(const nam_b200_model* m, double* out, int capacity);

/* Block until all work queued on the handle's stream has finished. */
int nam_b200_synchronize(nam_b200_model* m);

/* Number of kernels this handle has launched since creation (diagnostic, used by bench.py). */
int64_t nam_b200_launch_count(const nam_b200_model* m);

/* Device time of the most recent process_* / reset call's kernels in milliseconds (CUDA events on the
 * handle's stream); negative if unavailable. */
double nam_b200_last_kernel_ms(nam_b200_model* m);

/* Host-only: parse + validate a .nam document and describe what the library would do with it, as a
 * small JSON object written to `out` (NUL-terminated, truncated to `capacity`): architecture, channels,
 * prewarm_samples, n_weights, expected_sample_rate, flops_per_frame, state_bytes_per_stream,
 * kernel ("fused" | "lstm" | "linear" | "unsupported"), reason.  Never touches CUDA, so it is usable on a
 * machine without a GPU (host-logic tests).  Returns 0, or the same error codes as create. */
int nam_b200_inspect_json(const char* nam_json_text, int fast_tanh, char* out, int64_t capacity);
int nam_b200_inspect_file(const char* nam_path, int fast_tanh, char* out, int64_t capacity);

/* Host-only: build (or fetch from the cache) the model-specialised kernel of a WaveNet document without touching a
 * GPU -- NVRTC cross-compiles -- and describe the outcome as a small JSON object: ok, from_cache, compile_seconds,
 * cubin_bytes, threads, frames_per_thread, smem_bytes, why_not.  Used to pre-populate the cache at install time. */
int nam_b200_jit_prepare_json(const char* nam_json_text, int fast_tanh, char* out, int64_t capacity);
/* The same for the kernel geometry a handle of `max_batch` streams on a 132-SM device (H100 SXM) would get (the short-call entry point
 * packs 6, 7 or 8 streams per CTA, whichever fills whole waves best at max_batch). */
int nam_b200_jit_prepare_json_for_batch(const char* nam_json_text, int fast_tanh, int max_batch, char* out, int64_t capacity);
/* Diagnostic: how this handle's specialised kernel was obtained, or why it has none.  Returns the text's length. */
int64_t nam_b200_jit_note(const nam_b200_model* m, char* out, int64_t capacity);

/* Host-only: the sub-models of a slimmable document -- a "SlimmableContainer" file (NAM/container.cpp) or a WaveNet
 * whose layer arrays carry {"slimmable": {"method": "slice_channels_uniform"}} (NAM/wavenet/model.cpp:1290-1315,
 * NAM/wavenet/slimmable.cpp: one sliced plain WaveNet per interval between the ratio breakpoints).  index < 0: returns
 * the number of sub-models (0 = not slimmable).  Otherwise writes the sub-model's complete .nam document (truncated to
 * capacity - 1 bytes) and its max_value (nam_b200_set_slimmable_size picks the first sub-model with value <
 * max_value), and returns the document's full length. */
int64_t nam_b200_submodel_json(const char* nam_json_text, int index, double* max_value, char* out, int64_t capacity);

/* Thread-local message of the last failing call on this thread. */
const char* nam_b200_last_error(void);

/* Measured FP32 FMA issue rate of the device (FFMA micro-benchmark), in TFLOP/s.  Used by bench.py as the compute
 * roofline for the fused kernel.  `use_ffma2` is ignored: sm_90 has no packed FP32 FMA.  Returns < 0 on error. */
double nam_b200_measure_fp32_tflops(int device, int use_ffma2);

#ifdef __cplusplus
}
#endif
#endif /* NAM_B200_H */
