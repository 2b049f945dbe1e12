// wavenet_pack.h -- turn a WaveNetSpec into the weight blob + descriptors the fused kernel reads.
// Host only.  The layouts are documented in wavenet_fused.cuh (LayerDesc / ArrayDesc).
#pragma once

#include <string>
#include <vector>

#include "nam_model_spec.h"
#include "wavenet_desc.h"

namespace namb200
{

struct WaveNetPlan
{
  bool eligible = false;
  std::string why_not; // set when !eligible
  int n_arrays = 0;
  int cp[kMaxArrays] = {0, 0, 0, 0}; // padded channel count per array (4, 8 or 16)
  int creal[kMaxArrays] = {0, 0, 0, 0};
  std::vector<float> blob; // packed weights
  std::vector<ArrayDesc> arrays;
  std::vector<LayerDesc> layers;
  long state_floats = 0; // per-stream ring storage (floats), multiple of 32
  float head_scale = 1.0f;
  double macs_per_frame = 0.0; // algorithmic MACs (unpadded), for roofline reporting
  int max_lookback = 0;

  // tensor-core variant
};

/// Decide whether the fused kernel can run this model and, if so, pack it.
/// Eligible family (SURVEY.md section 8a "core"): mono in/out, no condition_dsp, no post-stack
/// head, 1 or 2 layer arrays, per array: condition_size 1, bottleneck == channels <= 16, groups 1,
/// layer1x1 active, no head1x1, no FiLM, gating "none", head kernel size 1.
WaveNetPlan plan_wavenet(const ModelSpec& ms);

} // namespace namb200
