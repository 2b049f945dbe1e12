// stream_state.cuh -- pack / unpack of per-stream state records (stream_state.h) and row copies between streams.
//
// One descriptor-driven kernel pair for every layout: the grid is (chunk of one segment's items) x (listed stream); a
// segment's descriptor (StateSegDesc) says how its columns sit in one stream's device state.  Ring column j (0 = oldest)
// of a stream whose history ends at clock t is at slot (t - lookback + j) & mask, correct across the wrap of the
// 32-bit clock.
//   plane rings [Cp/4][R][4]: an item is one (plane, column) float4; consecutive threads take consecutive columns of a
//     plane, so the ring reads (writes) coalesce except at the one wrap.  The record side is [column][Cr]; unpack writes
//     zeros into the pad channels, which the fused kernels rely on.
//   row rings [R][C]: an item is one float; a column is contiguous on both sides, a strided copy with one wrap.
//   flat: a straight copy.
// The kernels move bytes only (no arithmetic): bandwidth-bound.
#pragma once

#include "stream_state.h"

namespace namb200
{

struct StatePackParams
{
  const StateSegDesc* segs;
  const StateChunk* chunks;
  const float* state; // [stream][state_stride]
  const float* state_alt; // Linear: the other buffer of the double buffer (StreamRef::alt)
  long state_stride;
  const StreamRef* refs; // [n]
  int n;
  unsigned char* rec; // record i at rec + i * rec_stride
  long rec_stride;
  uint32_t header[kStateHeaderBytes / 4];
  const uint32_t* headers; // model bank: record s takes headers[refs[s].model] (kStateHeaderBytes each); nullptr: header
};

__global__ void __launch_bounds__(kStateThreads) state_pack_kernel(const __grid_constant__ StatePackParams p)
{
  const StateChunk ch = p.chunks[blockIdx.x];
  const StateSegDesc d = p.segs[ch.seg];
  const int i = ch.item0 + (int)threadIdx.x;
  for (int s = blockIdx.y; s < p.n; s += gridDim.y)
  {
    const StreamRef r = p.refs[s];
    unsigned char* rec = p.rec + (size_t)s * p.rec_stride;
    if (blockIdx.x == 0 && threadIdx.x < kStateHeaderBytes / 4)
      reinterpret_cast<uint32_t*>(rec)[threadIdx.x] =
        p.headers ? p.headers[(size_t)r.model * (kStateHeaderBytes / 4) + threadIdx.x] : p.header[threadIdx.x];
    if (i >= d.items)
      continue;
    const float* __restrict__ st = (r.alt ? p.state_alt : p.state) + (size_t)r.stream * p.state_stride + d.dev_off;
    float* __restrict__ out = reinterpret_cast<float*>(rec + kStateHeaderBytes) + d.canon_off;
    if (d.kind == kSegPlaneRing)
    {
      const int pl = i / d.lookback, col = i - pl * d.lookback;
      const uint32_t slot = (r.clock - (uint32_t)d.lookback + (uint32_t)col) & (uint32_t)d.mask;
      const float4 v = __ldcs(reinterpret_cast<const float4*>(st) + (size_t)pl * (d.mask + 1) + slot);
      float* o = out + (size_t)col * d.cr + 4 * pl;
      const int nc = d.cr - 4 * pl; // >= 1
      o[0] = v.x;
      if (nc > 1)
        o[1] = v.y;
      if (nc > 2)
        o[2] = v.z;
      if (nc > 3)
        o[3] = v.w;
    }
    else if (d.kind == kSegRowRing)
    {
      const int col = i / d.cr, c = i - col * d.cr;
      const uint32_t slot = (r.clock - (uint32_t)d.lookback + (uint32_t)col) & (uint32_t)d.mask;
      out[i] = __ldcs(st + (size_t)slot * d.cr + c);
    }
    else
      out[i] = st[i];
  }
}

struct StateUnpackParams
{
  const StateSegDesc* segs;
  const StateChunk* chunks;
  float* state;
  long state_stride;
  const StreamRef* refs;
  int n;
  const unsigned char* rec; // record i at rec + i * rec_stride (0: one record for every stream)
  long rec_stride;
};

__global__ void __launch_bounds__(kStateThreads) state_unpack_kernel(const __grid_constant__ StateUnpackParams p)
{
  const StateChunk ch = p.chunks[blockIdx.x];
  const StateSegDesc d = p.segs[ch.seg];
  const int i = ch.item0 + (int)threadIdx.x;
  if (i >= d.items)
    return;
  for (int s = blockIdx.y; s < p.n; s += gridDim.y)
  {
    const StreamRef r = p.refs[s];
    const float* __restrict__ in = reinterpret_cast<const float*>(p.rec + (size_t)s * p.rec_stride + kStateHeaderBytes) + d.canon_off;
    float* __restrict__ st = p.state + (size_t)r.stream * p.state_stride + d.dev_off;
    if (d.kind == kSegPlaneRing)
    {
      const int pl = i / d.lookback, col = i - pl * d.lookback;
      const uint32_t slot = (r.clock - (uint32_t)d.lookback + (uint32_t)col) & (uint32_t)d.mask;
      const float* src = in + (size_t)col * d.cr + 4 * pl;
      const int nc = d.cr - 4 * pl;
      const float4 v = make_float4(src[0], nc > 1 ? src[1] : 0.0f, nc > 2 ? src[2] : 0.0f, nc > 3 ? src[3] : 0.0f);
      reinterpret_cast<float4*>(st)[(size_t)pl * (d.mask + 1) + slot] = v;
    }
    else if (d.kind == kSegRowRing)
    {
      const int col = i / d.cr, c = i - col * d.cr;
      const uint32_t slot = (r.clock - (uint32_t)d.lookback + (uint32_t)col) & (uint32_t)d.mask;
      st[(size_t)slot * d.cr + c] = in[i];
    }
    else
      st[i] = in[i];
  }
}

// Whole rows of per-stream state: dst row (dst_refs ? dst_refs[i].stream : i) = src row (src_refs ? src_refs[i].stream : i),
// i < n.  stride4 = state floats per stream / 4 (every layout's stride is a multiple of 4 floats).
__global__ void __launch_bounds__(kStateThreads) state_rows_kernel(float4* __restrict__ dst, const float4* __restrict__ src,
                                                                    long stride4, const StreamRef* __restrict__ dst_refs,
                                                                    const StreamRef* __restrict__ src_refs, int n)
{
  const long k = (long)blockIdx.x * kStateThreads + threadIdx.x;
  if (k >= stride4)
    return;
  for (int i = blockIdx.y; i < n; i += gridDim.y)
  {
    const long ds = dst_refs ? dst_refs[i].stream : i, ss = src_refs ? src_refs[i].stream : i;
    dst[ds * stride4 + k] = src[ss * stride4 + k];
  }
}

} // namespace namb200
