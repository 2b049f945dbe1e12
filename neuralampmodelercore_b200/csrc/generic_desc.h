// generic_desc.h -- plain-data description of a WaveNet with the reference's full option set, shared by
// the host packer (generic_pack.cpp) and the general kernel (wavenet_generic.cuh).
//
// The fused kernels (wavenet_fused.cuh, wavenet_spec.cuh) cover the model families that matter for throughput
// (SURVEY.md 8a, 8f-1).  Everything else the reference's WaveNet can express -- gated / blended activations,
// bottleneck != channels, grouped convolutions, head1x1, the eight FiLM sites, a condition_dsp sub-model, the
// post-stack head (NAM/wavenet/model.cpp:19-103,183-393,777-910; NAM/film.h; NAM/gating_activations.h) -- runs
// through this description: every matrix dense (grouped ones are block diagonal with explicit zeros, which adds
// exact zeros to the sums); one CTA per stream, one thread per frame of a 128-frame tile, layer by layer.
#pragma once

#ifdef __CUDACC_RTC__ // (NVRTC: no system headers; the specialised general kernel includes this file)
typedef unsigned int uint32_t;
#else
#include <stdint.h>
#endif

namespace namb200
{

constexpr int kGenMaxVec = 64; // widest per-frame vector (channels, 2 x bottleneck, condition, head sizes)
constexpr int kGenMaxArrays = 4;
constexpr int kGenMaxHeadConvs = 8;
constexpr int kGenFilmSites = 8;
constexpr int kGenTile = 128; // frames per tile == threads per CTA of the general kernel

// y = W x (+ b): W stored transposed and padded, [in][out_pad] with out_pad = out rounded up to 4 (zeros), 16-byte
// aligned at weights[w_off]; b (out_pad floats, zero padded) at weights[b_off] or b_off < 0
struct GMat
{
  int in, out, w_off, b_off;
};

// causal dilated convolution; weights [k][in][out_pad] (as GMat, per tap), tap 0 = oldest.  The ring keeps the convolution's INPUT
// vectors of the last ring_mask + 1 >= look-back + kGenTile frames of a stream (a whole tile is written before
// any tap is read): element (slot, i) at float ring_off + slot * in + i of the stream's state
struct GConv
{
  int in, out, kernel, dilation, w_off, b_off, ring_off, ring_mask;
};

struct GAct
{
  int type; // ActType
  float p0, p1, p2, p3; // LeakyReLU slope | LeakyHardtanh min_val, max_val, min_slope, max_slope
  int slopes_off, n_slopes; // PReLU
};

struct GFilm
{
  int active, shift, dim;
  GMat css; // condition -> (shift ? 2 : 1) * dim, with bias
};

struct GLayer
{
  int channels, bottleneck, zrows, gating, has_l1x1, has_h1x1;
  GConv conv; // channels -> zrows
  GMat mixin; // condition -> zrows
  GMat l1x1; // bottleneck -> channels
  GMat h1x1; // bottleneck -> head1x1 out
  GAct act, sec;
  GFilm film[kGenFilmSites]; // FilmSite order (nam_model_spec.h)
};

struct GArray
{
  int input_size, channels, head_out_size, head_size, layer0, n_layers;
  GMat rechannel; // input_size -> channels, no bias
  GConv head; // head_out_size -> head_size (LayerArray head rechannel)
};

struct GNet
{
  int in_channels, out_channels, n_arrays, with_head, n_head_convs;
  float head_scale;
  GAct head_act;
  GArray arrays[kGenMaxArrays];
  GConv head_convs[kGenMaxHeadConvs]; // post-stack head (model.cpp:19-103)
};

// ConvNet (NAM/convnet.cpp): blocks of kernel-2 dilated convolution -> per-channel affine (folded BatchNorm, absent
// when bn_off < 0) -> activation, then a linear head
constexpr int kGenMaxBlocks = 48;
struct GConvNet
{
  int in_channels, out_channels, channels, n_blocks;
  GAct act;
  GMat head;
  GConv convs[kGenMaxBlocks];
  int bn_off[kGenMaxBlocks]; // weights[bn_off ..]: scale[channels] then loc[channels]; -1: no batchnorm
};

struct ConvNetKernelParams
{
  const float* weights;
  GConvNet net;
  float* state; // [stream][state_stride]
  long state_stride;
  const float* in; // stream s, channel c: in[s * in_stride + c * n_frames ..]
  float* out;
  long in_stride, out_stride;
  int batch, n_frames;
  uint32_t t_base;
  int n_weight_floats;
};

struct GenericKernelParams
{
  const float* weights;
  const GLayer* layers;
  GNet net;
  GNet cond; // condition_dsp sub-model (valid when has_cond)
  int has_cond;
  float* state; // [stream][state_stride]
  long state_stride; // floats
  const float* in;
  float* out;
  long in_stride, out_stride;
  int batch, n_frames;
  uint32_t t_base;
  int n_weight_floats; // multiple of 4; the kernel keeps the blob in shared memory when it was given the room
};

} // namespace namb200
