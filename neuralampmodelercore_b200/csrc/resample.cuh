// resample.cuh -- the kernels of the rate conversion around a model (nam_b200_options.resample; design in resample.h).
//
// A call of n host frames on a stream whose host-sample count since reset is h makes model samples
// k in [ceil(h L / M), ceil((h + n) L / M)) and returns host samples j in [h, h + n):
//   y[k]   = sum_i x[i] g_up[k M - i L]      (host -> model)
//   out[j] = sum_k z[k] g_dn[j L - k M]      (model -> host)
// Relative to the call, with c = (-h L) mod M (it depends on h mod M only), output o of either direction reads inputs
// r = floor((base + o A) / B) - shift - u, u = 0 .. T-1, with tap u of phase (base + o A) mod B:
//   host -> model: A = M, B = L, base = c,     shift = 0, inputs x (host frames), outputs y (model frames)
//   model -> host: A = L, B = M, base = M - c, shift = 1, inputs z (model frames), outputs out (host frames)
// Inputs before the call (r < 0) come from the stream's history of the direction's last T inputs per channel.
// Every output sample is one fmaf chain from the oldest tap to the newest, so the result does not depend on how a
// stream's audio is split into calls.
#pragma once

#include <cstdint>

namespace namb200
{

// one position of a converting call: its state row, c = (-h L) mod M, host frames n, model frames m
struct RsPos
{
  int stream, c, n, m;
};

constexpr int kRsMaxThreads = 256; // outputs per CTA (one per thread)
constexpr int kRsHistThreads = 128; // >= the longest history (kResampleMaxTaps)

struct ResampleParams
{
  const float* __restrict__ taps; // tap-major [T][B]
  int T, A, B;
  const RsPos* __restrict__ pos;
  int n_pos, group; // positions; positions per CTA (grid.x walks groups of them)
  const float* __restrict__ in; // position q, channel ch: in + q * in_stride + ch * in_pitch
  long in_stride;
  int in_pitch;
  float* __restrict__ out;
  long out_stride;
  int out_pitch;
  const float* __restrict__ hist; // state row s: hist + s * hist_stride + hist_off, channel ch's H columns oldest first
  int hist_stride, hist_off, H;
};

// grid (position groups, output tiles of blockDim.x, channels); dynamic shared memory: T*B taps + the input window
template <bool kUp>
__global__ void __launch_bounds__(kRsMaxThreads) resample_kernel(const __grid_constant__ ResampleParams p)
{
  extern __shared__ float smem[];
  float* st = smem;
  float* sx = smem + p.T * p.B;
  for (int i = threadIdx.x; i < p.T * p.B; i += blockDim.x)
    st[i] = __ldg(p.taps + i);
  const int ch = blockIdx.z;
  const int o0 = blockIdx.y * blockDim.x;
  const int shift = kUp ? 0 : 1;
  const int q1 = min((int)(blockIdx.x + 1) * p.group, p.n_pos);
  for (int q = blockIdx.x * p.group; q < q1; q++)
  {
    const RsPos r = p.pos[q];
    const int n_in = kUp ? r.n : r.m, n_out = kUp ? r.m : r.n;
    if (o0 >= n_out)
      continue; // (uniform over the CTA)
    const long long base = kUp ? r.c : p.B - r.c;
    const int o_last = min(o0 + (int)blockDim.x, n_out) - 1;
    const int r_lo = (int)((base + (long long)o0 * p.A) / p.B) - shift - (p.T - 1);
    const int r_hi = (int)((base + (long long)o_last * p.A) / p.B) - shift;
    const float* x = p.in + (size_t)q * p.in_stride + (size_t)ch * p.in_pitch;
    const float* h = p.hist + (size_t)r.stream * p.hist_stride + p.hist_off + (size_t)ch * p.H;
    __syncthreads(); // the taps are staged; the previous position's window is no longer read
    for (int w = threadIdx.x; w <= r_hi - r_lo; w += blockDim.x)
    {
      const int rr = r_lo + w;
      sx[w] = rr >= 0 ? (rr < n_in ? x[rr] : 0.0f) : h[p.H + rr];
    }
    __syncthreads();
    const int o = o0 + (int)threadIdx.x;
    if (o < n_out)
    {
      const long long v = base + (long long)o * p.A;
      const int vb = (int)(v / p.B);
      const int ph = (int)(v - (long long)vb * p.B);
      const float* xs = sx + (vb - shift - r_lo);
      float acc = 0.0f;
      for (int u = p.T - 1; u >= 0; u--)
        acc = fmaf(st[u * p.B + ph], xs[-u], acc);
      p.out[(size_t)q * p.out_stride + (size_t)ch * p.out_pitch + o] = acc;
    }
  }
}

struct ResampleHistoryParams
{
  const RsPos* __restrict__ pos;
  int in_channels; // rows [0, in_channels) of grid.y: the host -> model histories, the rest the model -> host ones
  const float* __restrict__ x; // the call's host input (as ResampleParams::in of the host -> model launch)
  long x_stride;
  int x_pitch;
  const float* __restrict__ z; // the model's output (as ResampleParams::in of the model -> host launch)
  long z_stride;
  int z_pitch;
  float* __restrict__ hist;
  int hist_stride, H_up, H_dn;
};

// After both conversions of a call: each listed stream's histories take the last H inputs of [history | this call].
// grid (positions, in_channels + out_channels), kRsHistThreads threads; a direction without new inputs is left alone.
__global__ void __launch_bounds__(kRsHistThreads) resample_history_kernel(const __grid_constant__ ResampleHistoryParams p)
{
  const RsPos r = p.pos[blockIdx.x];
  const bool up = (int)blockIdx.y < p.in_channels;
  const int ch = up ? blockIdx.y : blockIdx.y - p.in_channels;
  const int n = up ? r.n : r.m;
  if (n == 0)
    return;
  const int H = up ? p.H_up : p.H_dn;
  float* h = p.hist + (size_t)r.stream * p.hist_stride + (up ? 0 : p.in_channels * p.H_up) + (size_t)ch * H;
  const float* src = up ? p.x + (size_t)blockIdx.x * p.x_stride + (size_t)ch * p.x_pitch
                        : p.z + (size_t)blockIdx.x * p.z_stride + (size_t)ch * p.z_pitch;
  const int i = threadIdx.x;
  float v = 0.0f;
  if (i < H)
  {
    const int t = n - H + i;
    v = t >= 0 ? src[t] : h[i + n];
  }
  __syncthreads();
  if (i < H)
    h[i] = v;
}

// The resampler's part of a stream-state record, behind the model's payload at float `off`: resample_in (H_up columns of
// in_channels, oldest first), resample_out (H_dn columns of out_channels), resample_phase (h mod M, in refs[s].clock).
// Pack also writes header word 3 (L << 16 | M) and the payload float count.
struct ResampleRecordParams
{
  float* hist;
  int hist_stride, in_channels, out_channels, H_up, H_dn;
  const StreamRef* refs;
  int n;
  unsigned char* rec;
  long rec_stride, off;
  uint32_t ratio;
  uint64_t payload_floats;
};

__device__ __forceinline__ float* rs_record_hist(const ResampleRecordParams& p, int stream, int i)
{
  float* row = p.hist + (size_t)stream * p.hist_stride;
  const int nu = p.in_channels * p.H_up;
  if (i < nu)
    return row + (size_t)(i % p.in_channels) * p.H_up + i / p.in_channels;
  const int j = i - nu;
  return row + nu + (size_t)(j % p.out_channels) * p.H_dn + j / p.out_channels;
}

// grid (item chunks of 256, streams)
__global__ void __launch_bounds__(256) resample_pack_kernel(const __grid_constant__ ResampleRecordParams p)
{
  const int i = blockIdx.x * 256 + threadIdx.x;
  const int items = p.in_channels * p.H_up + p.out_channels * p.H_dn;
  for (int s = blockIdx.y; s < p.n; s += gridDim.y)
  {
    const StreamRef r = p.refs[s];
    unsigned char* rec = p.rec + (size_t)s * p.rec_stride;
    float* out = reinterpret_cast<float*>(rec + kStateHeaderBytes) + p.off;
    if (i == 0)
    {
      uint32_t* w = reinterpret_cast<uint32_t*>(rec);
      w[3] = p.ratio;
      w[4] = (uint32_t)(p.payload_floats & 0xffffffffu);
      w[5] = (uint32_t)(p.payload_floats >> 32);
      out[items] = (float)r.clock;
    }
    if (i < items)
      out[i] = *rs_record_hist(p, r.stream, i);
  }
}

__global__ void __launch_bounds__(256) resample_unpack_kernel(const __grid_constant__ ResampleRecordParams p)
{
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= p.in_channels * p.H_up + p.out_channels * p.H_dn)
    return;
  for (int s = blockIdx.y; s < p.n; s += gridDim.y)
  {
    const float* in = reinterpret_cast<const float*>(p.rec + (size_t)s * p.rec_stride + kStateHeaderBytes) + p.off;
    *rs_record_hist(p, p.refs[s].stream, i) = in[i];
  }
}

} // namespace namb200
