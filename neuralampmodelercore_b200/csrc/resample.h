// resample.h -- rational sample-rate conversion around a model (nam_b200_options.resample): the filter design and the
// polyphase tap tables, host-only.  The kernels that apply them are in resample.cuh.
//
// L / M = model_rate / host_rate reduced by their gcd.  One Kaiser-windowed sinc prototype g at the common rate host * L
// serves both directions: g_up = L * g (host -> model), g_dn = M * g (model -> host).  include/nam_b200.h gives the formula.
#pragma once

#include <string>
#include <vector>

namespace namb200
{

constexpr int kResampleMaxFactor = 1024; // L, M <= this
constexpr int kResampleMaxTaps = 128; // taps per output sample, either direction
constexpr double kResampleStopbandDb = 84.0; // Kaiser design attenuation (>= 80 dB measured on the float32 taps)

struct ResamplerDesign
{
  double host_rate = 0.0, model_rate = 0.0;
  int L = 1, M = 1; // model_rate / host_rate = L / M
  int n_taps = 0; // N, prototype length
  std::vector<float> g_up, g_dn; // L * g and M * g, rounded to float32, N each
  int taps_up = 0, taps_dn = 0; // taps per output sample: ceil(N / L), ceil(N / M)
  double latency_frames = 0.0; // group delay of both filters together, in host frames: (N - 1) / L
};

// The design for a host / model rate pair (true, *out), or false and *why.  Both rates must be integers in Hz, L, M <= 1024
// and the taps per output sample <= 128 in both directions; a refusal names both rates.
bool design_resampler(double host_rate, double model_rate, ResamplerDesign* out, std::string* why);

// One direction as the kernel reads it: tap-major [T][B], tap u of phase p = g[p + u * B] (0 past N), B = L for the
// host -> model direction, M for the other.
std::vector<float> resampler_phase_table(const std::vector<float>& g, int B, int T);

// The design as a JSON object (nam_b200_resampler_json).
std::string resampler_json(const ResamplerDesign& d);

} // namespace namb200
