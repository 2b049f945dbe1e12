// wavenet_desc.h -- plain-data descriptors shared by the host packer (wavenet_pack.cpp, compiled
// by the host compiler) and the fused kernel (wavenet_fused.cuh, compiled by nvcc).
#pragma once

#include <stdint.h>

#include "generic_desc.h" // StreamRef (jit_params.h)

namespace namb200
{

constexpr int kMaxLayers = 64;
constexpr int kMaxArrays = 4;
constexpr int kHalo = 64; // columns of left halo kept in the shared tile

// Activation codes follow ActType (nam_model_spec.h)
enum : int
{
  KACT_TANH = 0,
  KACT_HARDTANH = 1,
  KACT_FASTTANH = 2,
  KACT_RELU = 3,
  KACT_LEAKYRELU = 4,
  KACT_PRELU = 5,
  KACT_SIGMOID = 6,
  KACT_SILU = 7,
  KACT_HARDSWISH = 8,
  KACT_LEAKYHARDTANH = 9,
  KACT_SOFTSIGN = 10,
  KACT_IDENTITY = 100
};

struct LayerDesc
{
  int w_off; // float offset in the weight blob: conv[K][C][C] | b[C] | M[C] | P[C][C] | p[C] | slopes[C]
  int kernel, dilation;
  int lookback; // (K-1)*dilation
  int ring_off; // float offset of this layer's ring inside one stream's state: [C/4][R][4]
  int ring_mask; // R-1, R = power of two >= lookback
  int act;
  float ap0, ap1, ap2, ap3;
};

struct ArrayDesc
{
  int layer0, n_layers;
  int rech_off; // [CIN][C]
  int head_off; // [HK][C][HOUT] | bias[HOUT]
  // head rechannel = Conv1D over the head accumulator (model.cpp:397-400,548); kernel 1 in the classic models,
  // 16 in the A2 family.  HK > 1 keeps the last (HK-1)*dilation head columns of a stream in their own ring.
  int head_kernel, head_dilation;
  int head_ring_off, head_ring_mask;
};

struct WaveNetKernelParams
{
  const float* weights; // packed blob
  int n_weight_floats;
  float* state; // [batch][state_stride]
  long state_stride; // floats
  const float* in; // [batch][in_stride]
  float* out;
  long in_stride, out_stride;
  int batch, n_frames;
  uint32_t t_base; // absolute frame index of in[:,0] (mod 2^32)
  float head_scale;
  int n_arrays;
  ArrayDesc arrays[kMaxArrays];
  LayerDesc layers[kMaxLayers];
  // Tile-parallel mode (few streams, long calls): CTA b handles tile (b % tiles_per_stream) of stream
  // (b / tiles_per_stream) only; tile_flags[stream][tile] counts the ring hand-overs that tile has published
  // (one per layer, one per convolutional head), and tile c waits for tile c-1 at every step -- a wavefront over
  // (tile, layer) instead of a serial walk.  tile_flags == nullptr: the classic mode.
  int* tile_flags;
  int tiles_per_stream;
  // Lock-step variant of the tile-parallel mode (wavenet_fused_kernel<..., LS = true>): every tile writes ALL columns of
  // every layer's input into a per-call history buffer hist[stream][plane][hist_cols][4 floats] the moment it has
  // produced them and publishes the step right away, so tile c can start layer l as soon as tiles c-1 .. c-m have
  // finished layer l-1 (m = tiles the look-back spans): all tiles advance layer by layer together and a call costs
  // ~(layers) layer-steps instead of (tiles + layers).  The rings are only read during the call (history from before
  // the call) and rewritten from hist at the very end, once every tile of the stream has finished.
  float* hist; // [batch][hist_stride]
  long hist_stride; // floats per stream = total planes * hist_cols * 4
  int hist_cols; // tiles_per_stream * frames per tile
  int hist_plane0[kMaxArrays]; // first plane of array a: its layers' inputs, P planes each, then its head-conv input
  // low-latency kernel (wavenet_lat2.cuh): completion doorbell, a word of mapped host memory that receives done_seq once the
  // call's outputs are visible to the host (nullptr: none)
  unsigned* done_flag;
  unsigned done_seq;
  // slot table (nullptr: position b of the call is state row b, its history ending at t_base): position b uses state row
  // slots[b].stream, whose history ends at slots[b].clock.  Inputs, outputs, hist and tile flags stay indexed by position.
  const StreamRef* slots;
  // model bank (table calls only): position b runs model slots[b].model, whose blob is at weights + model * weight_stride
  // and whose output scale is head_scales[model].  head_scales == nullptr: one model (weights, head_scale).
  long weight_stride;
  const float* head_scales;
};

} // namespace namb200
