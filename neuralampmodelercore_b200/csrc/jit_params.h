// jit_params.h -- the parameter layouts of the model-specialised (NVRTC) kernels, shared by the host that launches them
// (nam_b200.cu) and the kernels (wavenet_spec.cuh, wavenet_lat.cuh, wavenet_generic_spec.cuh, lstm_spec.cuh).  jit_spec.cpp
// hands this file to NVRTC with every program, so host and device compile the same definitions.
#pragma once

#ifdef __CUDACC_RTC__ // (NVRTC: no system headers)
typedef unsigned int uint32_t;
#else
#include <stdint.h>
#endif

namespace namb200
{

// One stream of a launch that addresses streams through a table: the state row it uses and the clock at which that row's
// history ends.  The process kernels' slot tables (position i of the call -> slots[i]) and the pack / unpack launches of
// stream_state.cuh share it.
struct StreamRef
{
  int stream;
  uint32_t clock; // the handle clock at which the stream's history ends (pack, process) or will end (unpack)
  union
  {
    int alt; // Linear: the stream's history is in the alternate buffer of the double buffer
    int model; // fused WaveNet family and LSTM: the model of a bank (nam_b200_create_bank_*) this position runs; 0 otherwise
  };
  // process calls: frames this position runs, in [0, n_frames] of the launch (n_frames is the buffers' frame pitch).  A
  // position stops at its own count: frames past it are neither read nor written, and a stream with 0 keeps its state.
  // Pack / unpack launches ignore it.
  int frames;
};

// The single by-value parameter of wavenet_spec*_kernel, wavenet_generic_spec_kernel and the lstm_spec* kernels.
struct JitParams
{
  float* state; // [row][state_stride]
  long state_stride; // floats
  const float* in; // [batch][in_stride]
  float* out;
  long in_stride, out_stride;
  int batch, n_frames;
  uint32_t t_base; // absolute frame index of in[:, 0] (mod 2^32); the LSTM kernels have no clock and ignore it
  // slot table (nullptr: position b is state row b at t_base, running n_frames frames): position b uses row slots[b].stream
  // at slots[b].clock and runs slots[b].frames frames; inputs and outputs stay indexed by position
  const StreamRef* slots;
  // model bank (wavenet_generic_spec_kernel compiled for a bank's shape, gspec::bank): position b runs the blob at
  // weights + slots[b].model * weight_stride; every other kernel ignores these
  const float* weights;
  long weight_stride;
};

// wavenet_lat_kernel's parameter: the same, plus the completion doorbell (done_flag may be null): a word in mapped host
// memory that receives `seq` once every output of the call is visible to the host -- the host spins on it instead of
// paying a stream synchronisation per 64-frame call
struct LatParams : JitParams
{
  unsigned* done_flag;
  unsigned seq;
};

} // namespace namb200
