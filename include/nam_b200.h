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
  int32_t bank_capacity; /* models a bank can hold (nam_b200_create_bank_* only; every other create ignores it): 0 = the
                            number of documents it is created with; below that, or negative, is refused.  See the model
                            bank section */
  union
  {
    int32_t reserved[4]; /* the last four words, zero by default; code that zeroes reserved[0..3] keeps compiling and
                            keeps asking for the defaults */
    struct
    {
      int32_t resample; /* 0 (default) = the host rate given to nam_b200_reset is recorded and ignored, as by the
                           reference; 1 = convert every stream from that rate to the model's expected rate before the model
                           and back after it, on the device, in the same call (see the sample-rate conversion section).
                           Equal rates convert nothing: outputs and launches are then exactly those of 0.  Multi-GPU
                           handles refuse 1 */
      int32_t reserved_tail[3];
    };
  };
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
  int32_t resample_up, resample_down; /* L and M of the last reset's conversion (model / host = L / M); 1, 1 when none */
  int32_t resample_latency_frames; /* group delay of the conversion in host frames, rounded (0 when none) */
  int32_t reserved[2];
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

/* ---- per-stream state: reset, copy, export and import single streams ----------------------------------------------
 * A stream's state travels as a RECORD that does not depend on the handle's kernel, geometry or max_batch: a 64-byte
 * header -- magic "NAMS", uint32 format version 1, uint32 architecture (as nam_b200_info), uint32 0, uint64 payload float
 * count, uint64 model fingerprint (a hash of the architecture, the parsed config and the weight bits; fast_tanh and the
 * handle options are not part of it), zeros -- then the float32 payload, little-endian:
 *   WaveNet / ConvNet: per convolution with a look-back (K-1)*d > 0, in weight-stream order (the main network's layer
 *     convolutions and head convolutions, then a condition_dsp sub-model's), the last look-back columns of its input,
 *     oldest first, each column the real channel count;  LSTM: per layer h[H] then c[H];  Linear: the last
 *     receptive_field - 1 input samples, oldest first.
 * nam_b200_state_layout_json lists the segments.  A record can be stored per user session, moved to another handle of the
 * same model (any options) or to another GPU.  SlimmableContainer handles act on the active sub-model, whose fingerprint a
 * record carries: a record taken at one slimmable size is refused at another.
 *
 * The handle keeps, per stream, the clock value at which the stream's history ends.  A stream left out of process calls
 * (batch < max_batch, not listed in nam_b200_process_streams_f32, or given fewer frames than the longest row of a ragged
 * call) keeps its history at that older point: export reads it
 * there, and every process call that includes it again continues from its own clock -- a pause needs no export, import or
 * reset.  (Contiguous calls launch exactly as before while every stream in [0, batch) is in step with the handle; otherwise
 * they carry the per-stream clocks like nam_b200_process_streams_f32.)
 *
 * Stream lists hold indices in [0, max_batch); destinations must be distinct.  Everything is checked on the host before
 * anything runs (NAM_B200_ERR_INVALID_ARGUMENT with the offending stream and field; NAM_B200_ERR_STATE before reset). */

/* Bytes of one record (header + payload). */
int64_t nam_b200_stream_state_size(const nam_b200_model* m);
/* DSP::Reset for the listed streams only, with the last reset's settings (prewarm_on_reset, max_frames); every other stream is
 * untouched.  WaveNet / ConvNet / Linear: the state nam_b200_reset leaves (fresh is ignored).  LSTM: fresh = 0 keeps h, c and
 * prewarms on top of them, as nam_b200_reset does; fresh = 1 starts from the trained h0, c0 like a newly created handle. */
int nam_b200_reset_streams(nam_b200_model* m, const int32_t* streams, int n, int fresh);
/* dst[i] takes src[i]'s state (all sources are read before any destination is written: a swap works). */
int nam_b200_copy_streams(nam_b200_model* m, const int32_t* src, const int32_t* dst, int n);
/* Record of streams[i] -> dst + i * record_stride (record_stride >= nam_b200_stream_state_size).  Host memory, staged
 * through the device on the handle's stream; returns when the records are in `dst`. */
int nam_b200_export_streams(nam_b200_model* m, const int32_t* streams, int n, void* dst, int64_t record_stride);
/* Records src + i * record_stride -> streams[i] (whose histories then end at the handle's clock).  Host memory; every
 * header is checked before anything is copied; returns when done. */
int nam_b200_import_streams(nam_b200_model* m, const int32_t* streams, int n, const void* src, int64_t record_stride);
/* The same on device memory (4-byte aligned records), asynchronous on `cuda_stream` (NULL = the handle's stream).  The import
 * first copies the n headers (64 B each) to the host and checks them, synchronising `cuda_stream` once, before it launches. */
int nam_b200_export_streams_device(nam_b200_model* m, const int32_t* streams, int n, void* dst_device, int64_t record_stride,
                                   void* cuda_stream);
int nam_b200_import_streams_device(nam_b200_model* m, const int32_t* streams, int n, const void* src_device,
                                   int64_t record_stride, void* cuda_stream);
/* Host-only, no CUDA: the record of a .nam document as a JSON object -- architecture, header_bytes, payload_floats,
 * record_bytes, fingerprint, segments [{name, channels, columns, offset (floats into the payload)}].  A SlimmableContainer
 * describes its default (largest) sub-model.  Returns 0, or the error codes of create. */
int nam_b200_state_layout_json(const char* nam_json_text, char* out, int64_t capacity);

/* ---- model banks: one handle, streams of different captures of one architecture ----------------------------------------
 * A bank is a handle created from K >= 1 .nam documents of one shape; each of its max_batch streams is bound to one of the
 * K models, and every process call runs each listed stream with its own model's weights, in the launches an ordinary
 * handle's call of that batch takes.  Which documents can share a bank -- model 0 chooses one of four families:
 *   - WaveNets served by the fused kernel family (wavenet.nam, a1_standard, A2-Lite and A2-Full shapes); not
 *     SlimmableContainer files or slimmable WaveNets.  Models 1.. equal model 0 in everything
 *     but their weights: layer arrays, channels, kernel sizes, dilations, activations and their parameters, hence the
 *     packed kernel layout and blob length; the config object apart from its unused head_scale field (head_scale is the
 *     last weight, so it is per model); the expected sample rate.
 *   - WaveNets an ordinary handle serves with the general kernel (gating, FiLM, grouped convolutions, head1x1, bottleneck !=
 *     channels, a condition_dsp sub-model, a post-stack head, multi-channel in / out).  Models 1.. equal model 0 in the
 *     expected sample rate and prewarm length, every array and layer field (channels, bottleneck, kernel sizes, dilations,
 *     groups, gating mode, activations, FiLM sites, layer1x1 / head1x1), the post-stack head, the condition_dsp's shape,
 *     hence the general kernel's descriptors and blob length, and the config object.  Both output scales (the network's
 *     and the condition_dsp's head_scale) are weights, so they are per model; a nested condition_dsp document's weights,
 *     metadata and version are per model too.
 *   - ConvNets an ordinary handle serves.  Models 1.. equal model 0 in the sample rate, channels, dilations, BatchNorm
 *     presence, activation, in / out channels and the config object; the folded BatchNorm is per model.
 *   - LSTMs an ordinary handle serves (a model it would refuse is refused with its reason).  Models 1.. equal model 0 in
 *     the expected sample rate (hence the prewarm length), in_channels and out_channels, num_layers, input_size,
 *     hidden_size and the config object; their weights, trained h0 / c0 and head are per model.
 *   Linear and mixed families are refused: a WaveNet on the fused kernel with one on the general kernel (either order) is
 *   refused with "model k: kernel: ...", naming model 0's family.  Refusals (NAM_B200_ERR_UNSUPPORTED for a model outside
 *   the family, NAM_B200_ERR_MODEL for a mismatch) name the first offending model index and the field.  jit:
 *   - fused and LSTM banks: jit = 1 is refused (a model-specialised kernel compiles one model's weights into its code);
 *     jit = 0 or 3 silently keeps the precompiled kernels, and nam_b200_jit_note says so;
 *   - general-WaveNet banks: jit as on an ordinary handle, for the general kernel compiled for the bank's SHAPE (the
 *     descriptors are compiled in, each stream's weights are staged in shared memory; nam_b200_bank_jit_prepare_json):
 *     0 = default (on at max_batch >= 256), 1 = required (creation fails with the reason when it cannot be had, e.g. a
 *     blob over 200 KB), 2 = off, 3 = preferred.  jit_state and nam_b200_jit_note report it;
 *   - ConvNet banks: as an ordinary ConvNet handle (there is no compiled ConvNet kernel).
 *   kernel_geometry 4 (the general kernel) is refused for fused-family and LSTM banks; on a general-WaveNet bank it selects
 *   the precompiled general kernel (as on an ordinary handle), any other non-zero geometry is taken as 4, and a ConvNet bank
 *   ignores it as an ordinary ConvNet handle does.  A bank of one document and bank_capacity 0 or 1 is exactly
 *   nam_b200_create_from_json / _from_file, JIT included; with bank_capacity >= 2 it is a bank of K = 1 (precompiled
 *   kernels, table calls), so that models can be added to it.
 * Capacity: options.bank_capacity (0 = K) reserves room for that many models at creation; a value below K, or negative, is
 *   refused with NAM_B200_ERR_INVALID_ARGUMENT.  nam_b200_bank_add_models and _replace_model below never reallocate or
 *   move what live streams use.
 * All streams start bound to model 0.  Every call of this header works on a bank, each stream exactly (bit for bit) as the
 * same stream of an ordinary jit = 2 handle of its model:
 *   - process calls (nam_b200_process_f32 and _device, process_streams*, the ragged calls, the planar DSP::process on stream
 *     0, the pipelined host path): each stream runs its own model;
 *   - nam_b200_reset: a WaveNet stream ends in the prewarmed fresh state of its own model.  An LSTM keeps h, c across
 *     Reset: each stream is prewarmed in place with its own model (from h0 / c0 the first time, since creation writes every
 *     stream's h0 / c0);
 *   - nam_b200_prewarm: every stream is prewarmed from its current state with its own model;
 *   - reset_streams: a WaveNet stream, and an LSTM stream with fresh = 1, takes its current model's fresh state; an LSTM
 *     stream with fresh = 0 is prewarmed in place with its model;
 *   - copy_streams: the destination takes the source's model along with its state;
 *   - export_streams: a record carries the fingerprint of its stream's model;
 *   - import_streams: accepts a record of any model of the bank and binds the stream to it (with duplicate documents the
 *     lowest such index); a fingerprint outside the bank is refused, naming it.  A session therefore moves between a bank
 *     and an ordinary handle of its model in either direction;
 *   - nam_b200_set_fast_tanh: as on an ordinary handle (an LSTM bank rebuilds its model rows in the new regime before the
 *     next fresh-state copy).
 * Device memory, allocated at creation for C = bank_capacity models: C x (blob + 64-byte record header + model row) plus,
 * for fused-family WaveNets, C output scales, and a slot table of max(max_batch, C) 16-byte entries (LSTM: max_batch + C).
 * The C blobs (a1_standard: ~14k floats each; lstm.nam: 64 floats each; a general WaveNet's blob carries
 * its two output scales behind its weights, wavenet_a2_max: ~1.9k floats), and C "model rows" of state_stride floats
 * each (a1_standard: 196 KB each, so a capacity of 512 reserves ~130 MB; lstm.nam: 8 floats) that
 * hold every model's freshly reset state (an LSTM's: h0 / c0 plus the prewarm): reset prewarms them together -- an LSTM
 * bank in the same launches as its streams -- and reset_streams and assign_streams copy them (one launch whatever the mix).
 * Cost of mixing: an LSTM kernel's CTA holds several streams (lane groups: 128 / G of them; thread per stream: 64); the
 * lane-group kernel keeps one weight copy per distinct model of a CTA where they fit and makes another pass where they do
 * not, the thread-per-stream kernel makes one pass per distinct model (up to 64 with round-robin binding).  Keep a model's
 * streams in adjacent slots.  The general WaveNet and ConvNet kernels run one stream per CTA at a time: a CTA restages the
 * blob into shared memory only when its next stream's model differs. */
int nam_b200_create_bank_from_json(const char* const* texts, int n_models, const nam_b200_options* opts, nam_b200_model** out);
int nam_b200_create_bank_from_files(const char* const* paths, int n_models, const nam_b200_options* opts, nam_b200_model** out);
/* K of a bank; 1 for every other handle (so model index 0 is valid on every handle). */
int nam_b200_bank_size(const nam_b200_model* m);
/* bank_capacity of a bank (K when it was created with 0); 1 for every other handle. */
int nam_b200_bank_capacity(const nam_b200_model* m);
/* Growing a bank: the n documents take model indices K .. K + n - 1 (*first_index = K).  Each is parsed and checked against
 * model 0 exactly as nam_b200_create_bank_from_json does (same codes and wording; "model k" names the index the document
 * would receive); more than bank_capacity - K documents, or n < 1, is refused with NAM_B200_ERR_INVALID_ARGUMENT.  All or
 * nothing: every document is checked before any device work, and a refusal leaves the handle unchanged.  After a reset the
 * new model rows are prepared at once, each in the state nam_b200_reset would have left it in (current max_frames,
 * prewarm_on_reset, fast-tanh regime); only those rows are written -- no stream's state or clock changes and no existing
 * model row is recomputed.  Before the first reset they wait for it.  A general-WaveNet bank's shape-compiled kernel is
 * reused as it is (its cache key holds no weight).  Returns when the device work has finished; not real-time safe. */
int nam_b200_bank_add_models(nam_b200_model* m, const char* const* texts, int n, int32_t* first_index);
/* Recycling an index: model k takes another document of the bank's shape (checked as above): its blob, output scale,
 * record fingerprint, nam_b200_bank_model_info (and nam_b200_get_info for k = 0) and, after a reset, its model row.  Refused
 * with NAM_B200_ERR_STATE while any stream is bound to k (the message names how many and the lowest); move them with
 * nam_b200_assign_streams first.  The overwrite waits for every earlier call of the handle, on any CUDA stream, so an
 * asynchronous call still running model k finishes with the old weights.  Afterwards import refuses records of the old
 * document (unless another index still holds it) and accepts the new one's.  NAM_B200_ERR_UNSUPPORTED on a handle that is
 * not a bank.  Returns when done. */
int nam_b200_bank_replace_model(nam_b200_model* m, int k, const char* text);
/* Bind streams[i] to model models[i] and put it in the state of a freshly reset handle of that model (the reset_streams
 * contract, per model: for an LSTM, reset_streams with fresh = 1 on an ordinary handle of that model); every other stream
 * is untouched.  Checked on the host like the other stream lists (distinct streams in [0, max_batch), model indices in
 * [0, bank_size), after reset); a refusal names the entry.  On an ordinary handle, models all 0 is
 * nam_b200_reset_streams with fresh = 0 -- for an LSTM that keeps the running state and prewarms on top, unlike a bank,
 * which restarts the stream from its new model's h0 / c0. */
int nam_b200_assign_streams(nam_b200_model* m, const int32_t* streams, int n, const int32_t* models);
/* out[i] = the model streams[i] is bound to. */
int nam_b200_stream_models(const nam_b200_model* m, const int32_t* streams, int n, int32_t* out);
/* nam_b200_get_info with model k's document-level fields (loudness, input / output levels, expected sample rate, weight
 * count): what a server needs per capture for normalisation.  k = 0 on an ordinary handle is nam_b200_get_info. */
int nam_b200_bank_model_info(const nam_b200_model* m, int k, nam_b200_info* info);
/* Host-only, no CUDA: can these documents share a bank?  A JSON object: ok, n_models, reason (the first offending model
 * index and field; "" when ok), fingerprints (each parsed model's record fingerprint, an unsigned
 * 64-bit integer as in nam_b200_state_layout_json).  Returns 0 whatever
 * the verdict; NAM_B200_ERR_INVALID_ARGUMENT when the buffer is too small. */
int nam_b200_bank_check_json(const char* const* texts, int n_models, char* out, int64_t capacity);
/* Host-only, no CUDA: compile (or find in the cache) the general kernel compiled for the shape of a bank of general-kernel
 * WaveNets (the kernel such a bank runs under jit 0 / 1 / 3), as nam_b200_jit_prepare_json does for one model.  The cache
 * key holds no weight, so every bank of one shape shares the cubin.  A JSON object: ok, from_cache, compile_seconds,
 * cubin_bytes, threads, smem_bytes (one blob), why_not.  Refused like nam_b200_create_bank_from_json, and for every other
 * family with NAM_B200_ERR_UNSUPPORTED. */
int nam_b200_bank_jit_prepare_json(const char* const* texts, int n_models, int fast_tanh, char* out, int64_t capacity);

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

/* Streams streams[0..n) (distinct, in [0, max_batch), any order): row i of in / out belongs to streams[i]
 * (in + i*in_stride, channel planes back to back as in nam_b200_process_f32).  Each listed stream continues from its
 * own history, wherever its clock stands; unlisted streams are untouched.  Host pointers; returns when `out` is filled.
 * The kernel is the one a contiguous call of batch = n would get.  Afterwards each listed stream's clock, and the
 * handle's, has moved on by n_frames.  Everything is checked on the host before anything is queued (NAM_B200_ERR_STATE
 * before reset; NAM_B200_ERR_INVALID_ARGUMENT naming the stream or field); n == 0 or n_frames == 0 does nothing. */
int nam_b200_process_streams_f32(nam_b200_model* m, const int32_t* streams, int n, const float* in, float* out,
                                 int n_frames, int64_t in_stride, int64_t out_stride);
/* The same on device audio buffers, asynchronous on cuda_stream (NULL = the handle's stream).  `streams` is a host
 * array and may be reused as soon as the call returns. */
int nam_b200_process_streams_f32_device(nam_b200_model* m, const int32_t* streams, int n, const float* in_device,
                                        float* out_device, int n_frames, int64_t in_stride, int64_t out_stride,
                                        void* cuda_stream);

/* Ragged calls: like nam_b200_process_streams_f32, but row i runs its own number of frames, n_frames[i], in one launch.
 *   Layout: let n_max = max_i n_frames[i].  Row i belongs to streams[i]; channel c of row i is at
 *     in + i*in_stride + c*n_max, its valid frames are [0, n_frames[i]) and [n_frames[i], n_max) is padding -- a
 *     [n, channels, n_max] array maps directly.  `out` follows the same layout.  in_stride >= in_channels*n_max and
 *     out_stride >= out_channels*n_max.
 *   Padding: input padding is never read (NaN there changes nothing).  The device entry never writes output padding;
 *     the host entry writes zeros there, and its host buffers must span full rows, as for a nam_b200_process_streams_f32
 *     call of n_max frames.
 *   State and clocks: each listed stream continues from its own clock and advances by its own n_frames[i]; the handle's
 *     clock advances by n_max.  An entry of 0 is accepted: that stream's state and clock stay exactly as they were, the
 *     device entry does not touch its output row and the host entry zeros it.
 *   Checks: everything is checked on the host before anything is queued, as for nam_b200_process_streams_f32; in
 *     addition n_frames must not be NULL when n > 0 and each entry must lie in [0, max_frames] of the last reset (a
 *     refusal names the entry).  n == 0 or n_max == 0 does nothing.
 *   The kernel is the one a contiguous call of batch = n and n_frames = n_max would get; nam_b200_process_streams_f32 is
 *   this call with every count equal.  `streams` and `n_frames` are host arrays, reusable as soon as the call returns. */
int nam_b200_process_streams_ragged_f32(nam_b200_model* m, const int32_t* streams, int n, const int32_t* n_frames,
                                        const float* in, float* out, int64_t in_stride, int64_t out_stride);
/* The same on device audio buffers, asynchronous on cuda_stream (NULL = the handle's stream). */
int nam_b200_process_streams_ragged_f32_device(nam_b200_model* m, const int32_t* streams, int n, const int32_t* n_frames,
                                               const float* in_device, float* out_device, int64_t in_stride,
                                               int64_t out_stride, void* cuda_stream);

/* ---- sample-rate conversion (options.resample = 1) ----------------------------------------------------------------------
 * When nam_b200_reset gets a sample_rate other than the model's expected rate, every stream is converted from that host
 * rate to the model's rate before the model and back after it, on the device, in the same call.
 *   Rates: both must be integers in Hz.  L / M = model_rate / host_rate in lowest terms, L, M <= 1024, and the filter below
 *     must need at most 128 taps per output sample in each direction (rates within a factor of about 2.5: 44.1 <-> 48 kHz
 *     takes 58, 96 -> 48 kHz 107, 32 -> 48 kHz 80).  Otherwise, and when the expected rate is unknown (-1), reset fails with
 *     NAM_B200_ERR_INVALID_ARGUMENT naming both rates.  Equal rates convert nothing.
 *   Definition: let h be a stream's host-sample count since its last reset.  A call of n host frames makes model samples
 *     k in [ceil(h L / M), ceil((h + n) L / M)), y[k] = sum_i x[i] g_up[k M - i L], runs the model on them (z), and returns
 *     host samples j in [h, h + n), out[j] = sum_k z[k] g_dn[j L - k M].  Both sums are causal, so every call returns n
 *     frames and the result does not depend on how a stream's audio is split into calls (bit for bit: each output sample
 *     is one fixed-order fmaf chain).  It is scipy.signal.upfirdn(g_up, x, L, M), the model, then upfirdn(g_dn, z, M, L).
 *   Filter: one Kaiser-windowed sinc at the common rate fs = host_rate * L, designed in double precision and stored as
 *     float32, g_up = L g, g_dn = M g:  A = 84 dB, beta = 0.1102 (A - 8.7), fmin = min(host_rate, model_rate),
 *     fc = 0.45 fmin / fs, df = 0.1 fmin / fs (cycles per sample), N = ceil((A - 7.95) / (2.285 * 2 pi df)) + 1,
 *     g[n] = 2 fc sinc(2 fc (n - (N-1)/2)) I0(beta sqrt(1 - ((n - (N-1)/2) / ((N-1)/2))^2)) / I0(beta), n in [0, N),
 *     sinc(x) = sin(pi x) / (pi x).  Passband ripple <= 0.1 dB up to 0.4 fmin, stopband >= 80 dB from 0.5 fmin.  Taps per
 *     output: ceil(N / L) host -> model, ceil(N / M) model -> host.  Latency (both filters): (N - 1) / L host frames.
 *   max_frames of nam_b200_reset counts host frames; the model's own calls take up to ceil(max_frames L / M) frames, and
 *     prewarm runs at the model's rate on zeros in blocks of that size (the resampler histories stay zero).
 *   Every process entry converts: nam_b200_process_f32 and _device, process_streams*, the ragged calls (n_frames[i] are
 *     host frames; each stream advances its own h, and its model clock by its own count of model frames), the planar
 *     DSP::process on stream 0 (without the low-latency doorbell) and the host-buffer path (without its chunk pipeline).
 *     A stream left out of a call, or given 0 frames, keeps its resampler state and h.  A call runs the host -> model
 *     kernel, the model's launch (the ragged launch of n_max = the longest row's model frames; the contiguous one when
 *     every row has the same count and no table is needed), the model -> host kernel and one history update.
 *   State: reset_streams and assign_streams zero a stream's resampler histories and set h = 0; copy_streams carries them.
 *     A record of a converting handle appends three segments after the model's: resample_in (in_channels x ceil(N / L)
 *     columns, oldest first), resample_out (out_channels x ceil(N / M) columns), resample_phase (one float, h mod M); its
 *     header word 3 (bytes 12-15) holds L << 16 | M (0 on a handle that converts nothing).  Import refuses a record whose
 *     ratio differs from the handle's, naming the field.  nam_b200_stream_state_size therefore follows the last reset.
 *   Banks share one expected rate, hence one ratio; SlimmableContainer handles pass the option to their sub-models. */
/* Host-only, no CUDA: the conversion between these rates as a JSON object -- host_rate, model_rate, L, M, n_taps,
 * taps_per_output_up, taps_per_output_down, latency_frames (host frames, a double), g_up, g_dn (%.9g).  Refuses a pair
 * exactly as nam_b200_reset does (equal rates included: L = M = 1 is a valid design); NAM_B200_ERR_INVALID_ARGUMENT also
 * when the buffer is too small. */
int nam_b200_resampler_json(double host_rate, double model_rate, char* out, int64_t capacity);

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
