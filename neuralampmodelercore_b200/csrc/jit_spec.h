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
  int nt = 512; // threads per CTA
  int s = 1; // frames per thread
  int min_ctas = 2; // __launch_bounds__ second argument
  int short_streams = 8; // streams per CTA of the short-call entry point (64 frames each)
  int short128_streams = 4, short256_streams = 2; // ... of the entry points for calls of up to 128 / 256 frames
  int tile() const { return nt * s; }
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
  size_t smem_bytes() const { return (size_t)max_planes * (size_t)(staged_cols + geom.tile()) * 16; }
};

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
std::string generic_spec_header_source(const GenericPlan& gp);
SpecBuild build_generic_spec_kernel(const GenericPlan& gp);

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
