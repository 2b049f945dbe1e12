// jit_spec.h -- load-time specialisation of the fused WaveNet kernel (wavenet_spec.cuh) to ONE model.
//
// The reference builds a graph of Eigen objects per model at load time (NAM/wavenet/model.cpp:580-683); this library's
// throughput path goes one step further and compiles the model: NVRTC turns wavenet_spec.cuh + a generated header
// (layer table as constexpr data, weights as `__device__ const float[]`) into sm_90a SASS in which every weight is the
// immediate operand of an FFMA.  The cubin is cached on disk, keyed by a hash of everything that went into it.
// Host only; no CUDA runtime types in this header.
#pragma once

#include <string>
#include <vector>

#include "generic_pack.h"
#include "wavenet_pack.h"

namespace namb200
{

struct SpecGeometry
{
  int nt = 512; // threads per CTA == frames per tile (one frame per thread); build_spec_kernel: spec_tile_geometry
  int min_ctas = 2; // __launch_bounds__ second argument
  int short_streams = 8; // streams per CTA of the short-call entry point (64 frames each)
  int short128_streams = 4, short256_streams = 2; // ... of the entry points for calls of up to 128 / 256 frames
};

struct SpecBuild
{
  bool ok = false;
  std::string why_not; // !ok: the reason (not eligible / NVRTC missing / compile error + log)
  std::vector<char> cubin;
  std::vector<char> cubin_extra; // second program of the model (128- / 256-frame short-call entry points), may be empty
  SpecGeometry geom;
  int staged_cols = 0; // spec::LS: columns of history staged in front of the tile (max look-back of the model)
  int max_planes = 0; // widest array, in planes of 4 channels
  bool from_cache = false;
  bool has_short = false; // the cubin also holds wavenet_spec_short{,128,256}_kernel (several streams x 64 / 128 / 256 frames per CTA)
  double compile_seconds = 0.0;
  size_t smem_bytes() const { return (size_t)max_planes * (size_t)(staged_cols + geom.nt) * 16; }
};

/// The throughput kernel's tile for `plan` (g.nt, g.min_ctas): one 1024-thread CTA per SM when its history window and
/// tile fit in shared memory and the model does at least 512 FFMAs per thread and frame per history unit (layer or
/// convolutional head), else two 512-thread CTAs per SM.  A tile stages its stream's whole ring set and writes back its
/// newest columns, so 1024-frame tiles halve that traffic per frame, and one resident stream per SM keeps the resident
/// rings in half of L2 where two 512-thread CTAs per SM filled it.  But a single CTA per SM has no second CTA to fill its
/// barrier drains, so a model needs enough work between two barriers to come out ahead (H100: a1_standard, 640 FFMAs per
/// unit, +70%; a2_full, 483, -15%; DESIGN.md 2.1b).  Any model that fits two 512-thread CTAs per SM fits one of 1024.
void spec_tile_geometry(const WaveNetPlan& plan, SpecGeometry& g);

/// Can wavenet_spec.cuh serve this plan?  (The plan must already be eligible for the generic fused kernel.)
bool spec_eligible(const WaveNetPlan& plan, const SpecGeometry& g, std::string* why_not);

/// The generated model header (namespace spec).  Deterministic: the cache key hashes it.
std::string spec_header_source(const WaveNetPlan& plan);

/// Compile (or fetch from the disk cache) the specialised kernel for `plan`.
/// Cache directory: $NAM_B200_JIT_CACHE, else <directory of libnam_b200.so>/jit_cache.  Never throws.
SpecBuild build_spec_kernel(const WaveNetPlan& plan, const SpecGeometry& g);

/// The low-latency kernel (wavenet_lat.cuh: one CTA per stream, calls of up to 32 * frame_warps frames, output channels
/// split over four warp groups, all history requested at kernel start).  SpecBuild::geom.nt = threads per CTA,
/// lat_smem_bytes() = its dynamic shared memory.
size_t lat_smem_bytes(const WaveNetPlan& plan, int frames);
SpecBuild build_lat_kernel(const WaveNetPlan& plan, int frame_warps);

/// The general kernel (every WaveNet option of the reference) compiled for one model: wavenet_generic_spec.cuh with the
/// descriptors of generic_desc.h and the weights as constant data.  Entry point: wavenet_generic_spec_kernel, 128 threads.
/// bank = true: the kernel compiled for the SHAPE of a model bank's general WaveNets -- the descriptors as constants, no
/// weights: gspec::w(i) reads the current stream's blob (generic_bank_blob_floats floats: the weights, then the net's and
/// the condition_dsp's output scales) from dynamic shared memory, which the kernel stages when the stream's model changes.
/// The header holds no weight, so every bank of one shape shares one cubin.  Unavailable when a blob exceeds
/// kGenericBankSmemBytes.
std::string generic_spec_header_source(const GenericPlan& gp, bool bank = false);
SpecBuild build_generic_spec_kernel(const GenericPlan& gp, bool bank = false);
size_t generic_bank_blob_floats(const GenericPlan& gp);
constexpr size_t kGenericBankSmemBytes = 200 * 1024;

/// The same for a small mono LSTM (lstm_spec.cuh: one thread per stream, weights as FFMA immediates); the cubin holds
/// lstm_spec_kernel_exact and lstm_spec_kernel_fast (the fast-tanh switch is read at run time, lstm.cpp:48).
bool lstm_spec_eligible(const ModelSpec& ms, std::string* why_not);
std::string lstm_spec_header_source(const ModelSpec& ms);
SpecBuild build_lstm_spec_kernel(const ModelSpec& ms);

/// Name of the kernel entry point inside the cubin.
inline const char* spec_kernel_name()
{
  return "wavenet_spec_kernel";
}

} // namespace namb200
