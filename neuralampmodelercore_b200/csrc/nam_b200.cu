// nam_b200.cu -- C ABI of libnam_b200.so (include/nam_b200.h): model handles, device state,
// kernel launches.  Host code is C++; every hot-path operation is a hand-written sm_90a kernel
// (wavenet_fused.cuh, and the LSTM / Linear kernels below).  There is deliberately no CPU
// fallback anywhere in this file.
#include "../../include/nam_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <set>
#include <thread>
#include <string>
#include <vector>

#include "nam_model_spec.h"
#include "wavenet_fused.cuh"
#include "wavenet_lat2.cuh"
#include "wavenet_pack.h"
#include "generic_pack.h"
#include "wavenet_generic.cuh"
#include "jit_spec.h"

using namespace namb200;

// =================================================================================================
// error plumbing
// =================================================================================================
namespace
{
thread_local std::string g_last_error;

int fail(int code, const std::string& msg)
{
  g_last_error = msg;
  return code;
}

struct CudaError : public std::runtime_error
{
  using std::runtime_error::runtime_error;
};

#define CUDA_CHECK(expr)                                                                                             \
  do                                                                                                                 \
  {                                                                                                                  \
    cudaError_t _e = (expr);                                                                                         \
    if (_e != cudaSuccess)                                                                                           \
      throw CudaError(std::string(#expr) + " failed: " + cudaGetErrorString(_e));                                    \
  } while (0)

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device); safe when several handles launch from
// several host threads (the multi-device entry runs one worker thread per GPU)
void ensure_max_dynamic_smem(const void* kern, int device, int bytes)
{
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;
  std::lock_guard<std::mutex> lk(mu);
  if (done.count({kern, device}))
    return;
  CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.insert({kern, device});
}

// =================================================================================================
// LSTM kernel  (NAM/lstm.cpp:31-68 cell, :103-168 process)
//
// One THREAD per stream (the recurrence forbids parallelism over time, batch is the only
// parallel axis); the (W, b, head) parameters of all layers sit in shared memory and are read
// with warp-uniform broadcasts; each thread's (h, c) state lives in shared memory in
// [index][thread] order (conflict-free), is loaded from / stored to the per-stream state in
// global memory at launch boundaries.  Input/output frames are staged through shared memory
// in [32 streams x TC frames] tiles so global traffic is coalesced although each thread walks
// its own stream.
// =================================================================================================
struct LstmKernelParams
{
  const float* __restrict__ weights; // per layer: W[4H][I+H] | b[4H] ; then head_w[H] | head_b
  int n_weight_floats;
  float* __restrict__ state; // [batch][state_stride]: per layer h[H] | c[H]
  int state_stride;
  const float* __restrict__ in;
  float* __restrict__ out;
  long in_stride, out_stride;
  int batch, n_frames;
  int num_layers, input_size, hidden;
  int fast_tanh;
  // multi-channel models (lstm.cpp:103-125): stream b's channel c is the plane in[b * in_stride + c * n_frames ..];
  // input_size == in_channels.  Mono models take the staged (coalesced) path, in_ch == out_ch == 1.
  int in_ch, out_ch;
};

constexpr int kLstmThreads = 64; // streams per CTA
constexpr int kLstmChunk = 32; // frames staged per tile

__device__ __forceinline__ float lstm_sigmoid(float x, int fast)
{
  // fast regime: fast_sigmoid(x) = 0.5*(fast_tanh(x/2)+1)  (activations.h:100-103)
  return fast ? 0.5f * (act_fast_tanh(x * 0.5f) + 1.0f) : act_sigmoid(x);
}
__device__ __forceinline__ float lstm_tanh(float x, int fast)
{
  return fast ? act_fast_tanh(x) : tanhf(x);
}

__global__ void __launch_bounds__(kLstmThreads) lstm_kernel(const LstmKernelParams p)
{
  extern __shared__ float smem[];
  const int tid = threadIdx.x;
  const int H = p.hidden;
  float* sw = smem; // weights
  float* sstate = sw + ((p.n_weight_floats + 3) & ~3); // [num_layers*2*H][kLstmThreads]
  float* sgate = sstate + p.num_layers * 2 * H * kLstmThreads; // [4H][kLstmThreads] scratch
  float* sio = sgate + 4 * H * kLstmThreads; // [kLstmThreads][kLstmChunk+1] in, then same for out
  float* sout = sio + kLstmThreads * (kLstmChunk + 1);

  for (int i = tid; i < p.n_weight_floats; i += kLstmThreads)
    sw[i] = __ldg(p.weights + i);
  const int stream = blockIdx.x * kLstmThreads + tid;
  const bool active = stream < p.batch;
  const int n_state = p.num_layers * 2 * H;
  if (active)
    for (int i = 0; i < n_state; i++)
      sstate[i * kLstmThreads + tid] = p.state[(size_t)stream * p.state_stride + i];
  __syncthreads();

  const int stream0 = blockIdx.x * kLstmThreads;
  for (int t0 = 0; t0 < p.n_frames; t0 += kLstmChunk)
  {
    const int tc = min(kLstmChunk, p.n_frames - t0);
    // coalesced load of the [streams x tc] input tile
    for (int idx = tid; idx < kLstmThreads * kLstmChunk; idx += kLstmThreads)
    {
      const int s = idx / kLstmChunk, f = idx - s * kLstmChunk;
      float v = 0.0f;
      if (stream0 + s < p.batch && f < tc)
        v = __ldg(p.in + (size_t)(stream0 + s) * p.in_stride + t0 + f);
      sio[s * (kLstmChunk + 1) + f] = v;
    }
    __syncthreads();
    if (active)
    {
      const bool multi = p.in_ch > 1 || p.out_ch > 1;
      const float* __restrict__ gin = p.in + (size_t)stream * p.in_stride + t0;
      float* __restrict__ gout = p.out + (size_t)stream * p.out_stride + t0;
      for (int f = 0; f < tc; f++)
      {
        float x_scalar = sio[tid * (kLstmChunk + 1) + f];
        const float* w = sw;
        for (int l = 0; l < p.num_layers; l++)
        {
          const int I = (l == 0) ? p.input_size : H;
          const int W = I + H;
          float* hs = sstate + (l * 2) * H * kLstmThreads;
          float* cs = hs + H * kLstmThreads;
          const float* xprev = (l == 0) ? nullptr : sstate + ((l - 1) * 2) * H * kLstmThreads;
          const float* b = w + 4 * H * W;
          // ifgo = W [x ; h] + b   (lstm.cpp:36-40); rows ordered i, f, g, o
          for (int r = 0; r < 4 * H; r++)
          {
            const float* wr = w + r * W;
            float acc = 0.0f;
            if (l == 0 && !multi)
              acc = fmaf(wr[0], x_scalar, acc); // input_size == 1
            else if (l == 0)
              for (int j = 0; j < I; j++)
                acc = fmaf(wr[j], __ldg(gin + (size_t)j * p.n_frames + f), acc);
            else
              for (int j = 0; j < I; j++)
                acc = fmaf(wr[j], xprev[j * kLstmThreads + tid], acc);
            for (int j = 0; j < H; j++)
              acc = fmaf(wr[I + j], hs[j * kLstmThreads + tid], acc);
            sgate[r * kLstmThreads + tid] = acc + b[r];
          }
          for (int i = 0; i < H; i++)
          {
            const float gi = sgate[(i)*kLstmThreads + tid];
            const float gf = sgate[(H + i) * kLstmThreads + tid];
            const float gg = sgate[(2 * H + i) * kLstmThreads + tid];
            const float go = sgate[(3 * H + i) * kLstmThreads + tid];
            const float c = lstm_sigmoid(gf, p.fast_tanh) * cs[i * kLstmThreads + tid]
                            + lstm_sigmoid(gi, p.fast_tanh) * lstm_tanh(gg, p.fast_tanh); // lstm.cpp:50-53,61-63
            cs[i * kLstmThreads + tid] = c;
            hs[i * kLstmThreads + tid] = lstm_sigmoid(go, p.fast_tanh) * lstm_tanh(c, p.fast_tanh); // :55-57,65-66
          }
          w = b + 4 * H;
        }
        // head (lstm.cpp:164-167)
        const float* hl = sstate + ((p.num_layers - 1) * 2) * H * kLstmThreads;
        if (multi)
        {
          // head: (out_channels x H) row-major, then the bias vector (lstm.cpp:79-97)
          for (int oc = 0; oc < p.out_ch; oc++)
          {
            float y = 0.0f;
            for (int j = 0; j < H; j++)
              y = fmaf(w[oc * H + j], hl[j * kLstmThreads + tid], y);
            gout[(size_t)oc * p.n_frames + f] = y + w[p.out_ch * H + oc];
          }
          continue;
        }
        float y = 0.0f;
        for (int j = 0; j < H; j++)
          y = fmaf(w[j], hl[j * kLstmThreads + tid], y);
        sout[tid * (kLstmChunk + 1) + f] = y + w[H];
      }
    }
    __syncthreads();
    for (int idx = tid; idx < kLstmThreads * kLstmChunk; idx += kLstmThreads)
    {
      const int s = idx / kLstmChunk, f = idx - s * kLstmChunk;
      if (stream0 + s < p.batch && f < tc && p.out_ch == 1 && p.in_ch == 1)
        p.out[(size_t)(stream0 + s) * p.out_stride + t0 + f] = sout[s * (kLstmChunk + 1) + f];
    }
    __syncthreads();
  }
  if (active)
    for (int i = 0; i < n_state; i++)
      p.state[(size_t)stream * p.state_stride + i] = sstate[i * kLstmThreads + tid];
}

} // namespace
#include "lstm_group.cuh"
namespace
{

// =================================================================================================
// Linear (FIR) kernel, direct form (NAM/linear.cpp:168-199): y[t] = bias + sum_j w[j] x[t-j]
// One CTA per (stream, tile of frames); the tile plus RF-1 history samples are staged in shared
// memory; the per-stream history (last RF-1 samples) persists in global state.
// =================================================================================================
struct LinearKernelParams
{
  const float* __restrict__ impulse; // impulse[j] multiplies x[t-j]
  int rf;
  float bias;
  float* __restrict__ state; // [batch][state_stride]: last (rf-1) samples, oldest first
  int state_stride;
  const float* __restrict__ in;
  float* __restrict__ out;
  long in_stride, out_stride;
  int batch, n_frames;
};

constexpr int kLinThreads = 256;

__global__ void __launch_bounds__(kLinThreads) linear_kernel(const LinearKernelParams p)
{
  extern __shared__ float smem[];
  const int hist = p.rf - 1;
  float* sw = smem; // rf
  float* sx = smem + ((p.rf + 3) & ~3); // hist + kLinThreads
  const int stream = blockIdx.y;
  const int t0 = blockIdx.x * kLinThreads;
  const int tid = threadIdx.x;
  for (int i = tid; i < p.rf; i += kLinThreads)
    sw[i] = __ldg(p.impulse + i);
  const float* xin = p.in + (size_t)stream * p.in_stride;
  const float* st = p.state + (size_t)stream * p.state_stride;
  for (int i = tid; i < hist + kLinThreads; i += kLinThreads)
  {
    const int t = t0 - hist + i; // frame index relative to this call
    float v = 0.0f;
    if (t >= 0)
      v = (t < p.n_frames) ? __ldg(xin + t) : 0.0f;
    else
      v = st[hist + t]; // t in [-hist, 0): state holds frames -hist..-1
    sx[i] = v;
  }
  __syncthreads();
  const int t = t0 + tid;
  if (t < p.n_frames)
  {
    // oldest tap first, like the reference's dot over the reversed impulse (linear.cpp:71-74,184-186)
    float acc = 0.0f;
    for (int j = hist; j >= 0; j--)
      acc = fmaf(sw[j], sx[hist + tid - j], acc);
    p.out[(size_t)stream * p.out_stride + t] = p.bias + acc;
  }
}

// new_state = last (rf-1) samples of [old_state | in[0:n)]
__global__ void linear_update_state_kernel(const LinearKernelParams p, float* __restrict__ new_state)
{
  const int hist = p.rf - 1;
  const int stream = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= hist)
    return;
  const int t = p.n_frames - hist + i; // relative frame index of new history slot i
  float v;
  if (t >= 0)
    v = p.in[(size_t)stream * p.in_stride + t];
  else
    v = p.state[(size_t)stream * p.state_stride + hist + t];
  new_state[(size_t)stream * p.state_stride + i] = v;
}

// =================================================================================================
// misc kernels
// =================================================================================================
// Copy stream 0's state to streams [1, batch) (all streams are identical after prewarm).
__global__ void broadcast_state_kernel(float* __restrict__ state, long stride_floats, int batch)
{
  const long n4 = stride_floats / 4;
  const float4* src = reinterpret_cast<const float4*>(state);
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x)
  {
    const float4 v = src[i];
    for (int b = 1 + blockIdx.y; b < batch; b += gridDim.y)
      reinterpret_cast<float4*>(state + (size_t)b * stride_floats)[i] = v;
  }
}

// FP32 FMA issue-rate micro-benchmark: 8 independent accumulator pairs per thread (sm_90 has no packed FP32 FMA, so
// every pair is two scalar FFMAs).
__global__ void __launch_bounds__(256) fma_peak_kernel(float* out, int iters, float seed)
{
  float2 a[8];
#pragma unroll
  for (int i = 0; i < 8; i++)
    a[i] = make_float2(seed + i, seed - i);
  const float2 m = make_float2(1.0000001f, 0.9999999f);
  const float2 c = make_float2(1e-7f, -1e-7f);
  for (int it = 0; it < iters; it++)
  {
#pragma unroll
    for (int i = 0; i < 8; i++)
    {
      a[i].x = fmaf(a[i].x, m.x, c.x);
      a[i].y = fmaf(a[i].y, m.y, c.y);
    }
  }
  float s = 0.0f;
#pragma unroll
  for (int i = 0; i < 8; i++)
    s += a[i].x + a[i].y;
  if (s == 12345.678f)
    out[0] = s;
}

} // namespace

// =================================================================================================
// the handle
// =================================================================================================
struct nam_b200_model
{
  ModelSpec spec;
  nam_b200_options opts{};
  int device = 0;
  int sm_count = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  bool timing_valid = false;
  int64_t launches = 0;
  int max_frames = 0;
  bool is_reset = false;
  int reserved_sms = 0; // SMs the persistent throughput kernels leave free (nam_b200_set_reserved_sms)
  bool streams_identical = true; // every stream holds the same state (true after init_state, false once audio was processed)
  bool state_initialised = false; // init_state() has run at least once
  uint32_t t_base = 0;
  int fast_tanh_runtime = 0;

  // WaveNet
  WaveNetPlan plan;
  int variant = 0;
  int wn_ctas_per_sm = 0; // resident CTAs per SM of the fused kernel (occupancy query, cached)
  int* d_tile_flags = nullptr; // tile-parallel mode hand-over counters, one per resident CTA
  size_t tile_flags_capacity = 0;
  float* d_hist = nullptr; // lock-step tile-parallel mode: per-call history buffer (WaveNetKernelParams::hist)
  size_t hist_floats = 0;
  int wn_ctas_ls[3] = {0, 0, 0}; // resident CTAs per SM of the lock-step kernels (kLsGeom)
  int wn_ctas_short[2] = {0, 0}; // same for the short-call (multi-stream tile) geometries 2 / 3
  int wn_geometry = 1; // 0 / 1: index into kWnGeom (FFMA kernel)
  // model-specialised kernel (wavenet_spec.cuh compiled for this model by NVRTC, jit_spec.cpp): the throughput path
  cudaLibrary_t spec_lib = nullptr;
  cudaLibrary_t spec_lib_extra = nullptr; // second program of the model: the 128- / 256-frame short-call entry points
  cudaKernel_t spec_kernel = nullptr;
  struct SpecShort // its short-call entry points (q streams x fq frames per CTA; fq = 64, 128, 256), may be absent
  {
    cudaKernel_t kernel = nullptr;
    size_t smem = 0;
    int ctas_per_sm = 0, fq = 0, q = 0;
  } spec_short[3];
  cudaKernel_t gen_spec_kernel = nullptr; // wavenet_generic_spec.cuh: the general kernel compiled for this model
  cudaKernel_t lstm_spec_kernels[2] = {nullptr, nullptr}; // lstm_spec.cuh: exact / fast activation regime
  cudaKernel_t lstm_gate_kernels[2] = {nullptr, nullptr}; // its gate-split variant (four lanes per stream)
  // low-latency kernel (wavenet_lat.cuh): few streams x short calls; built by reset() for the handle's maxBufferSize
  cudaLibrary_t lat_lib = nullptr;
  cudaKernel_t lat_kernel = nullptr;
  int lat_frames = 0, lat_threads = 0; // calls of up to lat_frames frames
  size_t lat_smem = 0;
  int lat_state = 0; // like spec_state
  std::string lat_note;
  unsigned* h_flag = nullptr; // completion doorbell of the low-latency kernel: one word of mapped pinned memory
  unsigned* h_flag_dev = nullptr;
  unsigned flag_seq = 0;
  bool flag_pending = false; // the launch just issued rings the doorbell
  bool opts_timing_events = false; // $NAM_B200_TIMING=1: keep the per-call CUDA events (nam_b200_last_kernel_ms) on that path
  SpecGeometry spec_geom;
  size_t spec_smem = 0;
  int spec_ctas_per_sm = 0;
  int spec_state = 0; // 0 = not used, 1 = active, -1 = wanted but unavailable (spec_note says why)
  std::string spec_note;
  // general WaveNet kernel (wavenet_generic.cuh): every option the fused kernels do not specialise
  bool use_generic = false;
  GenericPlan gplan;
  GLayer* d_glayers = nullptr;
  // LSTM / Linear packed weights
  std::vector<float> host_weights;
  float* d_weights = nullptr;
  size_t n_weight_floats = 0;
  // per-stream state
  float* d_state = nullptr;
  float* d_state_tmp = nullptr; // Linear double buffer
  long state_stride = 0; // floats
  // staging
  float* d_in = nullptr;
  float* d_out = nullptr;
  size_t staging_floats = 0;
  float* h_pin = nullptr; // pinned, device-mapped scratch for the planar (single stream) entry points
  float* h_pin_dev = nullptr; // its device-side address
  size_t h_pin_floats = 0;
  double flops_per_frame = 0.0;

  // host-buffer calls on large batches are pipelined in chunks of streams: H2D(c+1) | kernel(c) | D2H(c-1)
  cudaStream_t copy_in = nullptr, copy_out = nullptr;
  std::vector<cudaEvent_t> chunk_events;

  // SlimmableContainer (NAM/container.cpp): the handle owns one complete sub-handle per sub-model and forwards
  // every call to the active one; it holds no device memory itself
  std::vector<std::unique_ptr<nam_b200_model>> subs;
  int active_sub = -1;
  double ext_sample_rate = -1.0;

  ~nam_b200_model()
  {
    cudaSetDevice(device);
    if (d_weights)
      cudaFree(d_weights);
    if (d_glayers)
      cudaFree(d_glayers);
    if (spec_lib)
      cudaLibraryUnload(spec_lib);
    if (spec_lib_extra)
      cudaLibraryUnload(spec_lib_extra);
    if (lat_lib)
      cudaLibraryUnload(lat_lib);
    if (d_tile_flags)
      cudaFree(d_tile_flags);
    if (d_hist)
      cudaFree(d_hist);
    if (d_state)
      cudaFree(d_state);
    if (d_state_tmp)
      cudaFree(d_state_tmp);
    if (d_in)
      cudaFree(d_in);
    if (d_out)
      cudaFree(d_out);
    if (h_pin)
      cudaFreeHost(h_pin);
    if (h_flag)
      cudaFreeHost(h_flag);
    if (ev0)
      cudaEventDestroy(ev0);
    if (ev1)
      cudaEventDestroy(ev1);
    for (cudaEvent_t e : chunk_events)
      cudaEventDestroy(e);
    if (copy_in)
      cudaStreamDestroy(copy_in);
    if (copy_out)
      cudaStreamDestroy(copy_out);
    if (stream)
      cudaStreamDestroy(stream);
  }
};

namespace
{

// ---- WaveNet launch dispatch -----------------------------------------------------------------
// Two CTA geometries of the same kernel (S = 2 time steps per thread):
//   geometry 0: 128 threads, tile 256 frames, >= 3 CTAs/SM (<= 168 registers)
//   geometry 1: 256 threads, tile 512 frames, >= 2 CTAs/SM (<= 128 registers) -- 16 warps/SM, the
//               weights (one copy per CTA) cost half the shared memory per warp
constexpr int kWnS = 2; // time steps per thread

//   geometry 2: 128 threads, the 256-frame tile split into 4 streams x 64 frames (short calls: the reference
//               tools' 64-frame blocks are latency-bound per stream, so 4 streams share a CTA's layer walk)
struct WnGeometry
{
  int nt, min_ctas, lq; // lq: log2(frames per sub-tile)
  int frames_per_subtile() const { return 1 << lq; }
  int streams_per_tile() const { return (kWnS * nt) >> lq; }
};
//   geometry 3: 256 threads, the 512-frame tile split into 4 streams x 128 frames (calls of 97..192 frames)
constexpr WnGeometry kWnGeom[4] = {{128, 3, 8}, {256, 2, 9}, {128, 3, 6}, {256, 2, 7}};
// calls of up to this many frames take the multi-stream geometry 2 / 3
constexpr int kWnShortMaxFrames[2] = {96, 192};

template <int C0, int C1, int NT, int MINB, int LQ>
void launch_wavenet_variant(nam_b200_model* m, const WaveNetKernelParams& kp, int grid, size_t smem, cudaStream_t st)
{
  auto kern = wavenet_fused_kernel<C0, C1, kWnS, NT, MINB, LQ>;
  ensure_max_dynamic_smem(reinterpret_cast<const void*>(kern), m->device, 227 * 1024);
  kern<<<grid, NT, smem, st>>>(kp);
  CUDA_CHECK(cudaGetLastError());
}

template <int C0, int C1, int NT, int MINB, int LQ>
int occupancy_wavenet_variant(size_t smem)
{
  auto kern = wavenet_fused_kernel<C0, C1, kWnS, NT, MINB, LQ>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  int n = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, NT, smem) != cudaSuccess)
    return 1;
  return n > 0 ? n : 1;
}

// lock-step tile-parallel kernels (LS = true), one stream per tile.
//   LS geometry 0: 128 threads x 2 frames, tile 256, >= 3 CTAs/SM  (default; kernel_geometry 1)
//   LS geometry 1: 256 threads x 2 frames, tile 512, >= 2 CTAs/SM  (kernel_geometry 2; also when tile 256 does not fit)
//   LS geometry 2: 128 threads x 1 frame, tile 128: only while every CTA has an SM to itself (batch x tiles <= SMs:
//                  one stream in 4096-frame calls), where a layer step is as long as one warp's instruction stream
// (A 256 x 1 geometry -- half the instructions per thread and layer step, twice the warps per tile -- doubles the weight
// loads per FMA.)
struct LsGeometry
{
  int nt, s, min_ctas, lq;
  int tile_frames() const { return 1 << lq; }
};
constexpr int kLsGeoms = 3;
constexpr LsGeometry kLsGeom[kLsGeoms] = {{128, 2, 3, 8}, {256, 2, 2, 9}, {128, 1, 3, 7}};

template <int C0, int C1, int S, int NT, int MINB, int LQ>
void launch_wavenet_ls_variant(nam_b200_model* m, const WaveNetKernelParams& kp, int grid, size_t smem, cudaStream_t st)
{
  auto kern = wavenet_fused_kernel<C0, C1, S, NT, MINB, LQ, true>;
  ensure_max_dynamic_smem(reinterpret_cast<const void*>(kern), m->device, 227 * 1024);
  // The tiles spin on each other's flags, so they must all be resident at once: a cooperative launch is
  // gang-scheduled (it starts only when the whole grid fits), which keeps two such launches from different handles
  // from starving each other.
  void* args[] = {const_cast<void*>(static_cast<const void*>(&kp))};
  CUDA_CHECK(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(kern), dim3((unsigned)grid), dim3(NT), args, smem, st));
}

template <int C0, int C1, int S, int NT, int MINB, int LQ>
int occupancy_wavenet_ls_variant(size_t smem)
{
  auto kern = wavenet_fused_kernel<C0, C1, S, NT, MINB, LQ, true>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  int n = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, NT, smem) != cudaSuccess)
    return 1;
  return n > 0 ? n : 1;
}

#define WN_LS_CASE(C0, C1, FN, ...)                                                                                  \
  case (C0) * 100 + (C1):                                                                                            \
    return geom == 0 ? FN<C0, C1, 2, 128, 3, 8>(__VA_ARGS__)                                                         \
                     : (geom == 1 ? FN<C0, C1, 2, 256, 2, 9>(__VA_ARGS__) : FN<C0, C1, 1, 128, 3, 7>(__VA_ARGS__));

#define WN_LS_DISPATCH(FN, ...)                                                                                      \
  switch (c0 * 100 + c1)                                                                                             \
  {                                                                                                                  \
    WN_LS_CASE(4, 0, FN, __VA_ARGS__)                                                                                \
    WN_LS_CASE(8, 0, FN, __VA_ARGS__)                                                                                \
    WN_LS_CASE(16, 0, FN, __VA_ARGS__)                                                                               \
    WN_LS_CASE(4, 4, FN, __VA_ARGS__)                                                                                \
    WN_LS_CASE(4, 8, FN, __VA_ARGS__)                                                                                \
    WN_LS_CASE(4, 16, FN, __VA_ARGS__)                                                                               \
    WN_LS_CASE(8, 4, FN, __VA_ARGS__)                                                                                \
    WN_LS_CASE(8, 8, FN, __VA_ARGS__)                                                                                \
    WN_LS_CASE(8, 16, FN, __VA_ARGS__)                                                                               \
    WN_LS_CASE(16, 4, FN, __VA_ARGS__)                                                                               \
    WN_LS_CASE(16, 8, FN, __VA_ARGS__)                                                                               \
    WN_LS_CASE(16, 16, FN, __VA_ARGS__)                                                                              \
    default: throw std::runtime_error("no fused WaveNet kernel for channel pair " + std::to_string(c0) + "/"         \
                                      + std::to_string(c1));                                                         \
  }

#define WN_CASE(C0, C1, FN, ...)                                                                                     \
  case (C0) * 100 + (C1):                                                                                            \
    return geom == 0 ? FN<C0, C1, 128, 3, 8>(__VA_ARGS__)                                                            \
                     : (geom == 1 ? FN<C0, C1, 256, 2, 9>(__VA_ARGS__)                                               \
                                  : (geom == 2 ? FN<C0, C1, 128, 3, 6>(__VA_ARGS__) : FN<C0, C1, 256, 2, 7>(__VA_ARGS__)));

#define WN_DISPATCH(FN, ...)                                                                                         \
  switch (c0 * 100 + c1)                                                                                             \
  {                                                                                                                  \
    WN_CASE(4, 0, FN, __VA_ARGS__)                                                                                   \
    WN_CASE(8, 0, FN, __VA_ARGS__)                                                                                   \
    WN_CASE(16, 0, FN, __VA_ARGS__)                                                                                  \
    WN_CASE(4, 4, FN, __VA_ARGS__)                                                                                   \
    WN_CASE(4, 8, FN, __VA_ARGS__)                                                                                   \
    WN_CASE(4, 16, FN, __VA_ARGS__)                                                                                  \
    WN_CASE(8, 4, FN, __VA_ARGS__)                                                                                   \
    WN_CASE(8, 8, FN, __VA_ARGS__)                                                                                   \
    WN_CASE(8, 16, FN, __VA_ARGS__)                                                                                  \
    WN_CASE(16, 4, FN, __VA_ARGS__)                                                                                  \
    WN_CASE(16, 8, FN, __VA_ARGS__)                                                                                  \
    WN_CASE(16, 16, FN, __VA_ARGS__)                                                                                 \
    default: throw std::runtime_error("no fused WaveNet kernel for channel pair " + std::to_string(c0) + "/"         \
                                      + std::to_string(c1));                                                         \
  }

void launch_wavenet_dispatch(int c0, int c1, int geom, nam_b200_model* m, const WaveNetKernelParams& kp, int grid,
                             size_t smem, cudaStream_t st)
{
  WN_DISPATCH(launch_wavenet_variant, m, kp, grid, smem, st)
}
int occupancy_wavenet_dispatch(int c0, int c1, int geom, size_t smem)
{
  WN_DISPATCH(occupancy_wavenet_variant, smem)
}

void launch_wavenet_ls_dispatch(int c0, int c1, int geom, nam_b200_model* m, const WaveNetKernelParams& kp, int grid,
                                size_t smem, cudaStream_t st)
{
  WN_LS_DISPATCH(launch_wavenet_ls_variant, m, kp, grid, smem, st)
}
int occupancy_wavenet_ls_dispatch(int c0, int c1, int geom, size_t smem)
{
  WN_LS_DISPATCH(occupancy_wavenet_ls_variant, smem)
}

// ---- few streams, short calls (the plugin protocol: one stream, 64-frame process() calls) ----------------------------
// Such a call is pure latency: ~22 layer steps, each as long as ONE warp needs for its frames' instructions.  A CTA
// of 128 threads x 1 frame (tile 128) halves the instructions per warp against the 2-frame geometries.
// ---- low-latency kernel (wavenet_lat2.cuh): one CTA per stream, calls of up to 64 / 128 frames --------------------------
size_t lat2_smem_bytes(const WaveNetPlan& plan, int F)
{
  int pmax = 0;
  for (int a = 0; a < plan.n_arrays; a++)
    pmax = std::max(pmax, plan.cp[a] / 4);
  size_t f4 = (plan.blob.size() + 3) / 4 + (size_t)2 * pmax * F;
  for (int a = 0; a < plan.n_arrays; a++)
    for (int i = 0; i < plan.arrays[a].n_layers; i++)
    {
      const LayerDesc& L = plan.layers[plan.arrays[a].layer0 + i];
      for (int k = 0; k + 1 < L.kernel; k++)
        f4 += (size_t)(plan.cp[a] / 4) * lat2_window_cols((L.kernel - 1 - k) * L.dilation, F);
    }
  return f4 * 16 + kMaxLayers * sizeof(int);
}
bool lat2_serves(const WaveNetPlan& plan, int F)
{
  for (int a = 0; a < plan.n_arrays; a++)
    if (plan.arrays[a].head_kernel != 1)
      return false;
  return plan.n_arrays <= 2 && lat2_smem_bytes(plan, F) <= 200 * 1024;
}
template <int C0, int C1>
void launch_wavenet_lat2_variant(nam_b200_model* m, const WaveNetKernelParams& kp, int fw, size_t smem, cudaStream_t st)
{
  if (fw == 2)
  {
    auto kern = wavenet_lat2_kernel<C0, C1, 2>;
    ensure_max_dynamic_smem(reinterpret_cast<const void*>(kern), m->device, 200 * 1024); // (+ 520 B of static mbarriers)
    kern<<<kp.batch, 256, smem, st>>>(kp);
  }
  else
  {
    auto kern = wavenet_lat2_kernel<C0, C1, 4>;
    ensure_max_dynamic_smem(reinterpret_cast<const void*>(kern), m->device, 200 * 1024);
    kern<<<kp.batch, 512, smem, st>>>(kp);
  }
  CUDA_CHECK(cudaGetLastError());
}
#define WN_LAT2_CASE(C0, C1) \
  case (C0) * 100 + (C1): return launch_wavenet_lat2_variant<C0, C1>(m, kp, fw, smem, st);
void launch_wavenet_lat2_dispatch(int c0, int c1, nam_b200_model* m, const WaveNetKernelParams& kp, int fw, size_t smem,
                                  cudaStream_t st)
{
  switch (c0 * 100 + c1)
  {
    WN_LAT2_CASE(4, 0) WN_LAT2_CASE(8, 0) WN_LAT2_CASE(16, 0) WN_LAT2_CASE(4, 4) WN_LAT2_CASE(4, 8) WN_LAT2_CASE(4, 16)
    WN_LAT2_CASE(8, 4) WN_LAT2_CASE(8, 8) WN_LAT2_CASE(8, 16) WN_LAT2_CASE(16, 4) WN_LAT2_CASE(16, 8) WN_LAT2_CASE(16, 16)
    default: throw std::runtime_error("no low-latency WaveNet kernel for channel pair " + std::to_string(c0) + "/" + std::to_string(c1));
  }
}

constexpr int kSmallNt = 128, kSmallLq = 7;
template <int C0, int C1>
void launch_wavenet_small_variant(nam_b200_model* m, const WaveNetKernelParams& kp, int grid, size_t smem, cudaStream_t st)
{
  auto kern = wavenet_fused_kernel<C0, C1, 1, kSmallNt, 3, kSmallLq, false>;
  ensure_max_dynamic_smem(reinterpret_cast<const void*>(kern), m->device, 227 * 1024);
  kern<<<grid, kSmallNt, smem, st>>>(kp);
  CUDA_CHECK(cudaGetLastError());
}
#define WN_SMALL_CASE(C0, C1) \
  case (C0) * 100 + (C1): return launch_wavenet_small_variant<C0, C1>(m, kp, grid, smem, st);
void launch_wavenet_small_dispatch(int c0, int c1, nam_b200_model* m, const WaveNetKernelParams& kp, int grid, size_t smem,
                                   cudaStream_t st)
{
  switch (c0 * 100 + c1)
  {
    WN_SMALL_CASE(4, 0) WN_SMALL_CASE(8, 0) WN_SMALL_CASE(16, 0) WN_SMALL_CASE(4, 4) WN_SMALL_CASE(4, 8) WN_SMALL_CASE(4, 16)
    WN_SMALL_CASE(8, 4) WN_SMALL_CASE(8, 8) WN_SMALL_CASE(8, 16) WN_SMALL_CASE(16, 4) WN_SMALL_CASE(16, 8) WN_SMALL_CASE(16, 16)
    default: throw std::runtime_error("no fused WaveNet kernel for channel pair " + std::to_string(c0) + "/" + std::to_string(c1));
  }
}
size_t wavenet_small_smem_bytes(const WaveNetPlan& plan)
{
  const int cmax = std::max(plan.cp[0], plan.cp[1]);
  return (plan.blob.size() + 3) / 4 * 16 + (size_t)(cmax / 4) * (kHalo + (1 << kSmallLq)) * 16;
}

size_t wavenet_ls_smem_bytes(const WaveNetPlan& plan, int g)
{
  const int cmax = std::max(plan.cp[0], plan.cp[1]);
  return (plan.blob.size() + 3) / 4 * 16 + (size_t)(cmax / 4) * (kHalo + kLsGeom[g].tile_frames()) * 16;
}

// ---- lock-step tile-parallel mode: geometry choice and history buffer -----------------------------------------------
// planes (4 channels each) of hist per stream: every layer's input, plus the head accumulator of a convolutional head
int wavenet_hist_planes(const WaveNetPlan& plan, int* plane0 = nullptr)
{
  int planes = 0;
  for (int a = 0; a < plan.n_arrays; a++)
  {
    if (plane0)
      plane0[a] = planes;
    planes += (plan.arrays[a].n_layers + (plan.arrays[a].head_kernel > 1 ? 1 : 0)) * (plan.cp[a] / 4);
  }
  return planes;
}

// resident CTAs of the lock-step kernel of LS geometry g on the whole device; 0 if it cannot run
long wavenet_ls_capacity(nam_b200_model* m, int g)
{
  const WaveNetPlan& plan = m->plan;
  const size_t smem = wavenet_ls_smem_bytes(plan, g);
  if (smem > 227 * 1024)
    return 0;
  if (m->wn_ctas_ls[g] <= 0)
    m->wn_ctas_ls[g] = occupancy_wavenet_ls_dispatch(plan.cp[0], plan.n_arrays > 1 ? plan.cp[1] : 0, g, smem);
  return (long)m->wn_ctas_ls[g] * m->sm_count;
}

// is LS geometry g a candidate under the handle's options?  kernel_geometry 1 / 2 pin LS geometry 0 / 1; the default
// tries 0 (tile 256) and then 1 (tile 512: half as many CTAs to keep co-resident)
bool wavenet_ls_candidate(const nam_b200_model* m, int g)
{
  if (g == 2)
    return m->opts.kernel_geometry == 0; // (chosen first, and only while batch x tiles <= SMs: wavenet_ls_geometry)
  return m->opts.kernel_geometry == 0 || g == m->opts.kernel_geometry - 1;
}

// The LS geometry the lock-step mode would use for (batch, n_frames): the first candidate whose CTAs are all
// co-resident, -1 if none.
int wavenet_ls_geometry(nam_b200_model* m, int batch, int n_frames, int* tiles_out)
{
  if (m->opts.tile_mode != 0 || m->use_generic)
    return -1;
  static const int order[kLsGeoms] = {2, 0, 1};
  for (int oi = 0; oi < kLsGeoms; oi++)
  {
    const int g = order[oi];
    if (!wavenet_ls_candidate(m, g))
      continue;
    const int tf = kLsGeom[g].tile_frames();
    const int tiles = (n_frames + tf - 1) / tf;
    const long cap = (g == 2) ? std::min<long>(wavenet_ls_capacity(m, g), m->sm_count) : wavenet_ls_capacity(m, g);
    if (tiles >= 2 && (long)batch * tiles <= cap)
    {
      *tiles_out = tiles;
      return g;
    }
  }
  return -1;
}

// reset(): size the history buffer and the flags for every (batch <= max_batch, n_frames <= max_frames) the
// lock-step mode can serve, so that process() never allocates
void ensure_hist(nam_b200_model* m)
{
  if (m->spec.arch != Arch::WaveNet || m->use_generic || m->opts.tile_mode != 0)
    return;
  const int planes = wavenet_hist_planes(m->plan);
  size_t need = 0, need_flags = 0;
  for (int g = 0; g < kLsGeoms; g++)
  {
    if (!wavenet_ls_candidate(m, g))
      continue;
    const int tf = kLsGeom[g].tile_frames();
    const long tiles_max = (m->max_frames + tf - 1) / tf;
    const long cap = (g == 2) ? std::min<long>(wavenet_ls_capacity(m, g), m->sm_count) : wavenet_ls_capacity(m, g);
    if (tiles_max < 2 || cap < 2)
      continue;
    const long ctas = std::min<long>((long)m->opts.max_batch * tiles_max, cap);
    need = std::max(need, (size_t)ctas * tf * planes * 4);
    need_flags = std::max(need_flags, (size_t)ctas);
  }
  if (need > m->hist_floats)
  {
    if (m->d_hist)
      cudaFree(m->d_hist);
    m->d_hist = nullptr;
    m->hist_floats = 0;
    CUDA_CHECK(cudaMalloc(&m->d_hist, need * sizeof(float)));
    m->hist_floats = need;
  }
  if (need_flags > m->tile_flags_capacity)
  {
    if (m->d_tile_flags)
      cudaFree(m->d_tile_flags);
    m->d_tile_flags = nullptr;
    m->tile_flags_capacity = 0;
    CUDA_CHECK(cudaMalloc(&m->d_tile_flags, need_flags * sizeof(int)));
    m->tile_flags_capacity = need_flags;
  }
}

size_t wavenet_smem_bytes(const WaveNetPlan& plan, int geom)
{
  const int cmax = std::max(plan.cp[0], plan.cp[1]);
  const WnGeometry& g = kWnGeom[geom];
  const size_t tile4 = (size_t)(cmax / 4) * g.streams_per_tile() * (kHalo + g.frames_per_subtile());
  return (plan.blob.size() + 3) / 4 * 16 + tile4 * 16;
}

// ---- tensor-core variant dispatch ---------------------------------------------------------------
// `stream0`: index of the handle's stream that d_in / d_out row 0 belongs to (chunked host calls)
// ---- model-specialised kernel (wavenet_spec.cuh, compiled per model by jit_spec.cpp) ----------------------------------
// Mirror of namb200_spec::SpecParams (wavenet_spec.cuh): the kernel's single by-value parameter.
struct SpecKernelParams
{
  float* state;
  long state_stride;
  const float* in;
  float* out;
  long in_stride, out_stride;
  int batch, n_frames;
  uint32_t t_base;
  float* scratch; // stream-pair variant (S = 2) only: per-CTA interleaved rings; the shipped geometry is S = 1
  long scratch_stride;
};

int jit_mode(const nam_b200_model* m);

struct GenSpecKernelParams // mirror of namb200_gspec::GParams
{
  float* state;
  long state_stride;
  const float* in;
  float* out;
  long in_stride, out_stride;
  int batch, n_frames;
  unsigned t_base;
};


// Geometry of the specialised kernel for a handle of `max_batch` streams.  Streams per CTA of the short-call entry point:
// the count that fills whole waves of 2 CTAs per SM best (4096 streams on 132 SMs: 8 per CTA = 512 CTAs = 1.94 waves, 7 per
// CTA = 586 = 2.22 waves).
SpecGeometry spec_geometry_for(int max_batch, int sm_count)
{
  SpecGeometry g;
  double best = -1.0;
  auto pick = [&](std::initializer_list<int> candidates, int& streams) {
    best = -1.0;
    for (int q : candidates)
    {
      const double slots = (max_batch + q - 1) / q, resident = 2.0 * sm_count;
      const double eff = slots / (std::ceil(slots / resident) * resident);
      if (eff > best + 0.02)
      {
        best = eff;
        streams = q;
      }
    }
  };
  pick({8, 7, 6}, g.short_streams);
  pick({4, 3}, g.short128_streams);
  g.short256_streams = 2;
  return g;
}

// Decide whether this handle gets a specialised kernel, build / fetch it, load it.  jit option: 0 = auto (on for
// throughput handles: max_batch >= 256, where one compilation pays for itself within the first calls), 1 = required
// (creation fails with the reason if it cannot be had), 2 = off.  $NAM_B200_JIT=0/1 overrides "auto".
void setup_spec_kernel(nam_b200_model* m)
{
  const int mode = jit_mode(m);
  const bool wanted = mode == 1 || ((mode == 0 || mode == 3) && m->opts.max_batch >= 256);
  if (!wanted || m->opts.kernel_geometry != 0)
    return;
  const SpecGeometry g = spec_geometry_for(m->opts.max_batch, m->sm_count);
  SpecBuild b = build_spec_kernel(m->plan, g);
  if (!b.ok)
  {
    m->spec_state = -1;
    m->spec_note = b.why_not;
    if (mode == 1)
      throw std::runtime_error("model-specialised kernel unavailable: " + b.why_not);
    return;
  }
  auto check = [&](cudaError_t e, const char* what) {
    if (e != cudaSuccess)
      throw CudaError(std::string(what) + " failed: " + cudaGetErrorString(e));
  };
  try
  {
    check(cudaLibraryLoadData(&m->spec_lib, b.cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0), "cudaLibraryLoadData");
    check(cudaLibraryGetKernel(&m->spec_kernel, m->spec_lib, spec_kernel_name()), "cudaLibraryGetKernel");
    m->spec_geom = b.geom;
    m->spec_smem = b.smem_bytes();
    check(cudaFuncSetAttribute((const void*)m->spec_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)m->spec_smem),
          "cudaFuncSetAttribute(spec kernel)");
    int occ = 0;
    check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (const void*)m->spec_kernel, b.geom.nt, m->spec_smem),
          "cudaOccupancyMaxActiveBlocksPerMultiprocessor(spec kernel)");
    if (occ < 1)
      throw CudaError("the specialised kernel does not fit on an SM");
    m->spec_ctas_per_sm = occ;
    if (b.has_short)
    {
      const char* const names[3] = {"wavenet_spec_short_kernel", "wavenet_spec_short128_kernel", "wavenet_spec_short256_kernel"};
      const int fqs[3] = {64, 128, 256}, qs[3] = {b.geom.short_streams, b.geom.short128_streams, b.geom.short256_streams};
      if (!b.cubin_extra.empty()
          && cudaLibraryLoadData(&m->spec_lib_extra, b.cubin_extra.data(), nullptr, nullptr, 0, nullptr, nullptr, 0) != cudaSuccess)
        m->spec_lib_extra = nullptr;
      for (int v = 0; v < 3; v++)
      {
        nam_b200_model::SpecShort& sv = m->spec_short[v];
        sv = nam_b200_model::SpecShort{};
        cudaLibrary_t lib = (v == 0) ? m->spec_lib : m->spec_lib_extra;
        if (lib == nullptr || cudaLibraryGetKernel(&sv.kernel, lib, names[v]) != cudaSuccess)
        {
          sv.kernel = nullptr;
          continue;
        }
        sv.fq = fqs[v];
        sv.q = qs[v];
        sv.smem = (size_t)b.max_planes * sv.fq * sv.q * 16;
        if (cudaFuncSetAttribute((const void*)sv.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sv.smem) != cudaSuccess
            || cudaOccupancyMaxActiveBlocksPerMultiprocessor(&sv.ctas_per_sm, (const void*)sv.kernel, sv.fq * sv.q, sv.smem)
                 != cudaSuccess
            || sv.ctas_per_sm < 1)
          sv.kernel = nullptr;
      }
    }
    cudaGetLastError();
    m->spec_state = 1;
    m->spec_note = b.from_cache ? "cubin from cache" : "compiled in " + std::to_string(b.compile_seconds) + " s";
  }
  catch (const CudaError& ex)
  {
    if (m->spec_lib)
      cudaLibraryUnload(m->spec_lib);
    if (m->spec_lib_extra)
      cudaLibraryUnload(m->spec_lib_extra);
    m->spec_lib = m->spec_lib_extra = nullptr;
    for (auto& sv : m->spec_short)
      sv = nam_b200_model::SpecShort{};
    m->spec_kernel = nullptr;
    m->spec_state = -1;
    m->spec_note = ex.what();
    if (mode == 1)
      throw;
  }
}

// the handle's JIT mode with the environment override applied: 1 required, 2 off, 3 preferred (try, fall back silently),
// 0 automatic
int jit_mode(const nam_b200_model* m)
{
  int mode = m->opts.jit;
  if (mode == 0 || mode == 3)
  {
    const char* e = std::getenv("NAM_B200_JIT");
    if (e && *e)
      mode = (e[0] == '0') ? 2 : (mode == 3 ? 3 : 1);
  }
  return mode;
}

struct LatKernelParams // mirror of namb200_lat::LatParams
{
  float* state;
  long state_stride;
  const float* in;
  float* out;
  long in_stride, out_stride;
  int batch, n_frames;
  uint32_t t_base;
  unsigned* done_flag;
  unsigned seq;
};

// reset(): plugin-style handles (few streams, maxBufferSize <= 128) get the low-latency kernel for calls of up to
// 64 / 128 frames.  Wanted when jit is "required" or "preferred" (the C++ shim's default), never by the automatic policy.
void setup_lat_kernel(nam_b200_model* m)
{
  if (m->spec.arch != Arch::WaveNet || m->use_generic || m->opts.kernel_geometry != 0)
    return;
  const int mode = jit_mode(m);
  if (!(mode == 1 || mode == 3) || m->opts.max_batch > m->sm_count || m->max_frames > 128)
    return;
  const int fw = m->max_frames <= 64 ? 2 : 4;
  if (m->lat_state == 1 && m->lat_frames == 32 * fw)
    return;
  if (m->lat_lib)
    cudaLibraryUnload(m->lat_lib);
  m->lat_lib = nullptr;
  m->lat_kernel = nullptr;
  m->lat_state = 0;
  SpecBuild b = build_lat_kernel(m->plan, fw);
  if (!b.ok)
  {
    m->lat_state = -1;
    m->lat_note = b.why_not;
    return; // the precompiled short-call geometries serve the handle
  }
  cudaError_t e = cudaLibraryLoadData(&m->lat_lib, b.cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
  if (e == cudaSuccess)
    e = cudaLibraryGetKernel(&m->lat_kernel, m->lat_lib, "wavenet_lat_kernel");
  m->lat_smem = lat_smem_bytes(m->plan, 32 * fw);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute((const void*)m->lat_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)m->lat_smem);
  if (e != cudaSuccess)
  {
    cudaGetLastError();
    if (m->lat_lib)
      cudaLibraryUnload(m->lat_lib);
    m->lat_lib = nullptr;
    m->lat_kernel = nullptr;
    m->lat_state = -1;
    m->lat_note = std::string("loading the low-latency kernel failed: ") + cudaGetErrorString(e);
    return;
  }
  if (!m->h_flag && cudaHostAlloc(&m->h_flag, 64, cudaHostAllocMapped) == cudaSuccess)
  {
    *m->h_flag = 0;
    if (cudaHostGetDevicePointer(&m->h_flag_dev, m->h_flag, 0) != cudaSuccess)
      m->h_flag_dev = nullptr;
  }
  cudaGetLastError();
  m->lat_frames = 32 * fw;
  m->lat_threads = b.geom.nt;
  m->lat_state = 1;
  m->lat_note = b.from_cache ? "cubin from cache" : "compiled in " + std::to_string(b.compile_seconds) + " s";
}

void launch_wavenet_lat(nam_b200_model* m, const WaveNetKernelParams& kp, cudaStream_t st)
{
  // single-stream calls ring the doorbell in mapped host memory (process_planar spins on it instead of synchronising)
  unsigned* flag = (kp.batch == 1 && m->h_flag_dev != nullptr) ? m->h_flag_dev : nullptr;
  if (flag)
    m->flag_seq++;
  LatKernelParams lp{kp.state, kp.state_stride, kp.in, kp.out, kp.in_stride, kp.out_stride, kp.batch, kp.n_frames, kp.t_base,
                     flag, m->flag_seq};
  m->flag_pending = flag != nullptr;
  void* args[] = {&lp};
  CUDA_CHECK(cudaLaunchKernel((const void*)m->lat_kernel, dim3(kp.batch), dim3(m->lat_threads), args, m->lat_smem, st));
}

void launch_wavenet_spec(nam_b200_model* m, const WaveNetKernelParams& kp, cudaStream_t st)
{
  SpecKernelParams sp{kp.state, kp.state_stride, kp.in,  kp.out, kp.in_stride, kp.out_stride,
                      kp.batch, kp.n_frames,     kp.t_base, nullptr, 0};
  void* args[] = {&sp};
  int grid = std::min(kp.batch, m->spec_ctas_per_sm * std::max(1, m->sm_count - m->reserved_sms));
  if (grid < 1)
    grid = 1;
  CUDA_CHECK(cudaLaunchKernel((const void*)m->spec_kernel, dim3(grid), dim3(m->spec_geom.nt), args, m->spec_smem, st));
}

void launch_wavenet(nam_b200_model* m, const float* d_in, float* d_out, int batch, int n_frames, long in_stride,
                    long out_stride, cudaStream_t st, int stream0 = 0)
{
  if (m->use_generic && m->gen_spec_kernel != nullptr && m->opts.kernel_geometry == 0)
  {
    GenSpecKernelParams sp{m->d_state + (size_t)stream0 * (size_t)m->state_stride, m->state_stride, d_in, d_out, in_stride, out_stride,
                           batch, n_frames, m->t_base};
    void* args[] = {&sp};
    CUDA_CHECK(cudaLaunchKernel((const void*)m->gen_spec_kernel, dim3(std::max(1, std::min(batch, 16 * m->sm_count))), dim3(kGenTile),
                                args, 0, st));
    m->launches++;
    return;
  }
  if (m->use_generic)
  {
    GenericKernelParams gp{};
    gp.weights = m->d_weights;
    gp.layers = m->d_glayers;
    gp.net = m->gplan.net;
    gp.cond = m->gplan.cond;
    gp.has_cond = m->gplan.has_cond ? 1 : 0;
    gp.state = m->d_state + (size_t)stream0 * (size_t)m->state_stride;
    gp.state_stride = m->state_stride;
    gp.in = d_in;
    gp.out = d_out;
    gp.in_stride = in_stride;
    gp.out_stride = out_stride;
    gp.batch = batch;
    gp.n_frames = n_frames;
    gp.t_base = m->t_base;
    gp.n_weight_floats = (int)((m->n_weight_floats + 3) & ~(size_t)3);
    const size_t wbytes = (size_t)gp.n_weight_floats * sizeof(float);
    const int grid_g = std::min(batch, 16 * m->sm_count);
    if (wbytes <= 200 * 1024)
    {
      ensure_max_dynamic_smem(reinterpret_cast<const void*>(wavenet_generic_kernel<true>), m->device, 200 * 1024);
      wavenet_generic_kernel<true><<<grid_g, kGenTile, wbytes, st>>>(gp);
    }
    else
      wavenet_generic_kernel<false><<<grid_g, kGenTile, 0, st>>>(gp);
    CUDA_CHECK(cudaGetLastError());
    m->launches++;
    return;
  }
  const WaveNetPlan& plan = m->plan;
  WaveNetKernelParams kp{};
  kp.weights = m->d_weights;
  kp.n_weight_floats = (int)plan.blob.size();
  kp.state = m->d_state + (size_t)stream0 * (size_t)m->state_stride;
  kp.state_stride = m->state_stride;
  kp.in = d_in;
  kp.out = d_out;
  kp.in_stride = in_stride;
  kp.out_stride = out_stride;
  kp.batch = batch;
  kp.n_frames = n_frames;
  kp.t_base = m->t_base;
  kp.head_scale = plan.head_scale;
  kp.n_arrays = plan.n_arrays;
  for (size_t i = 0; i < plan.arrays.size(); i++)
    kp.arrays[i] = plan.arrays[i];
  for (size_t i = 0; i < plan.layers.size(); i++)
    kp.layers[i] = plan.layers[i];
  const int geom = m->wn_geometry;
  const int c0 = plan.cp[0], c1 = plan.n_arrays > 1 ? plan.cp[1] : 0;
  // few streams, short calls: the precompiled low-latency kernel (wavenet_lat2.cuh): one CTA per stream, the weight blob and
  // every history window of the call brought in by bulk copies at kernel start ($NAM_B200_LAT_KERNEL=jit: prefer the
  // model-specialised wavenet_lat.cuh where the handle has it, =off: neither)
  {
    const char* lat_env = std::getenv("NAM_B200_LAT_KERNEL"); // (read per call: tests switch it)
    // 0: the model-specialised kernel where the handle has it, else the precompiled one (both faster than the 128 x 1
    // geometry they replace); "precompiled" / "jit" / "off" pin the choice
    const int lat_pref = !lat_env ? 0 : (std::strcmp(lat_env, "jit") == 0 ? 1 : (std::strcmp(lat_env, "off") == 0 ? 2 : (std::strcmp(lat_env, "precompiled") == 0 ? 3 : 0)));
    const int fw = n_frames <= 64 ? 2 : 4;
    const bool jit_lat_ok = lat_pref != 2 && lat_pref != 3 && m->lat_state == 1 && n_frames <= m->lat_frames && batch <= m->sm_count;
    if (!jit_lat_ok && lat_pref != 1 && lat_pref != 2 && m->opts.kernel_geometry == 0 && n_frames <= 128 && batch <= m->sm_count
        && lat2_serves(plan, 32 * fw))
    {
      if (batch == 1 && m->h_flag_dev != nullptr)
      {
        kp.done_flag = m->h_flag_dev;
        kp.done_seq = ++m->flag_seq;
        m->flag_pending = true;
      }
      launch_wavenet_lat2_dispatch(c0, c1, m, kp, fw, lat2_smem_bytes(plan, 32 * fw), st);
      m->launches++;
      return;
    }
    if (jit_lat_ok)
    {
      // the model-specialised variant (wavenet_lat.cuh)
      launch_wavenet_lat(m, kp, st);
      m->launches++;
      return;
    }
  }
  // short calls on many streams, specialised: q streams x 64 / 128 / 256 frames per CTA (wavenet_spec_short*_kernel)
  if (m->spec_state == 1 && m->opts.kernel_geometry == 0 && n_frames <= 256)
    for (const nam_b200_model::SpecShort& sv : m->spec_short)
    {
      if (n_frames > sv.fq)
        continue;
      if (sv.kernel == nullptr || batch < 2 * sv.q)
        break; // the smallest variant that holds the call, or none
      {
        SpecKernelParams sp{kp.state, kp.state_stride, kp.in,  kp.out, kp.in_stride, kp.out_stride,
                            kp.batch, kp.n_frames,     kp.t_base, nullptr, 0};
        void* args[] = {&sp};
        const int grid_s = std::max(1, std::min((batch + sv.q - 1) / sv.q, sv.ctas_per_sm * m->sm_count));
        CUDA_CHECK(cudaLaunchKernel((const void*)sv.kernel, dim3(grid_s), dim3(sv.fq * sv.q), args, sv.smem, st));
        m->launches++;
        return;
      }
    }
  // short calls on more than a handful of streams: several streams per tile (same rings, same arithmetic)
  for (int sg = 0; sg < 2; sg++)
  {
    const int g = 2 + sg;
    if (n_frames > kWnShortMaxFrames[sg])
      continue;
    if (batch < 2 * kWnGeom[g].streams_per_tile() || wavenet_smem_bytes(plan, g) > 227 * 1024 || m->opts.kernel_geometry != 0)
      break;
    const size_t smem_s = wavenet_smem_bytes(plan, g);
    if (m->wn_ctas_short[sg] <= 0)
      m->wn_ctas_short[sg] = occupancy_wavenet_dispatch(c0, c1, g, smem_s);
    const int q = kWnGeom[g].streams_per_tile();
    const int grid_s = std::min((batch + q - 1) / q, m->wn_ctas_short[sg] * m->sm_count);
    launch_wavenet_dispatch(c0, c1, g, m, kp, std::max(grid_s, 1), smem_s, st);
    m->launches++;
    return;
  }
  // few streams (every CTA alone on its SM), short calls: the 128 x 1 geometry
  if (m->opts.kernel_geometry == 0 && n_frames <= (1 << kSmallLq) && batch <= m->sm_count
      && wavenet_small_smem_bytes(plan) <= 227 * 1024)
  {
    launch_wavenet_small_dispatch(c0, c1, m, kp, batch, wavenet_small_smem_bytes(plan), st);
    m->launches++;
    return;
  }
  const size_t smem = wavenet_smem_bytes(plan, geom);
  if (m->wn_ctas_per_sm <= 0)
  {
    const int occ = occupancy_wavenet_dispatch(c0, c1, geom, smem);
    // (a user value above the real occupancy would overstate co-residency for the spin-waiting tile-parallel launches)
    m->wn_ctas_per_sm = m->opts.ctas_per_sm > 0 ? std::min(m->opts.ctas_per_sm, std::max(occ, 1)) : occ;
  }
  const int per_sm = m->wn_ctas_per_sm;
  // Few streams, long calls, lock-step: one CTA per (stream, tile), all tiles advancing layer by layer together
  // (WaveNetKernelParams::hist).  All CTAs must be co-resident.
  {
    int tiles = 0;
    const int g = wavenet_ls_geometry(m, batch, n_frames, &tiles);
    if (g >= 0)
    {
      const int tf = kLsGeom[g].tile_frames();
      int plane0[kMaxArrays] = {0, 0, 0, 0};
      const int planes = wavenet_hist_planes(plan, plane0);
      const size_t per_stream = (size_t)planes * tiles * tf * 4;
      if ((size_t)batch * per_stream <= m->hist_floats && (size_t)batch * tiles <= m->tile_flags_capacity)
      {
        CUDA_CHECK(cudaMemsetAsync(m->d_tile_flags, 0, (size_t)batch * tiles * sizeof(int), st));
        kp.tile_flags = m->d_tile_flags;
        kp.tiles_per_stream = tiles;
        kp.hist = m->d_hist;
        kp.hist_stride = (long)per_stream;
        kp.hist_cols = tiles * tf;
        for (int a = 0; a < kMaxArrays; a++)
          kp.hist_plane0[a] = plane0[a];
        launch_wavenet_ls_dispatch(c0, c1, g, m, kp, batch * tiles, wavenet_ls_smem_bytes(plan, g), st);
        m->launches++;
        return;
      }
    }
  }
  // The same as a wavefront (tile_mode 1): a tile hands its ring columns to its successor layer by layer, so tile c
  // runs one layer behind tile c-1 -- (tiles + layers) layer-steps per call, but no history buffer.
  if (m->opts.tile_mode == 1)
  {
    const int tile_frames = kWnS * kWnGeom[geom].nt;
    const int tiles = (n_frames + tile_frames - 1) / tile_frames;
    const long capacity = (long)per_sm * m->sm_count;
    if (tiles >= 2 && (long)batch * tiles <= capacity && 2L * batch <= capacity)
    {
      if ((size_t)capacity > m->tile_flags_capacity)
      {
        if (m->d_tile_flags)
          cudaFree(m->d_tile_flags);
        m->d_tile_flags = nullptr;
        m->tile_flags_capacity = 0;
        CUDA_CHECK(cudaMalloc(&m->d_tile_flags, (size_t)capacity * sizeof(int)));
        m->tile_flags_capacity = (size_t)capacity;
      }
      CUDA_CHECK(cudaMemsetAsync(m->d_tile_flags, 0, (size_t)batch * tiles * sizeof(int), st));
      kp.tile_flags = m->d_tile_flags;
      kp.tiles_per_stream = tiles;
      launch_wavenet_dispatch(c0, c1, geom, m, kp, batch * tiles, smem, st);
      m->launches++;
      return;
    }
  }
  if (m->spec_state == 1 && m->opts.kernel_geometry == 0)
  {
    launch_wavenet_spec(m, kp, st);
    m->launches++;
    return;
  }
  int grid = std::min(batch, per_sm * std::max(1, m->sm_count - m->reserved_sms));
  if (grid < 1)
    grid = 1;
  launch_wavenet_dispatch(c0, c1, geom, m, kp, grid, smem, st);
  m->launches++;
}

// ---- model-specialised LSTM kernel (lstm_spec.cuh through jit_spec.cpp): same policy as setup_spec_kernel ------------
struct LstmSpecKernelParams // mirror of namb200_lstm_spec::LstmSpecParams
{
  float* state;
  long state_stride;
  const float* in;
  float* out;
  long in_stride, out_stride;
  int batch, n_frames;
};

void setup_lstm_spec_kernel(nam_b200_model* m)
{
  const int mode = jit_mode(m);
  if (!(mode == 1 || ((mode == 0 || mode == 3) && m->opts.max_batch >= 256)))
    return;
  SpecBuild b = build_lstm_spec_kernel(m->spec);
  if (!b.ok)
  {
    m->spec_state = -1;
    m->spec_note = b.why_not;
    if (mode == 1)
      throw std::runtime_error("model-specialised kernel unavailable: " + b.why_not);
    return;
  }
  auto check = [&](cudaError_t e, const char* what) {
    if (e != cudaSuccess)
      throw CudaError(std::string(what) + " failed: " + cudaGetErrorString(e));
  };
  try
  {
    check(cudaLibraryLoadData(&m->spec_lib, b.cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0), "cudaLibraryLoadData");
    check(cudaLibraryGetKernel(&m->lstm_spec_kernels[0], m->spec_lib, "lstm_spec_kernel_exact"), "cudaLibraryGetKernel");
    check(cudaLibraryGetKernel(&m->lstm_spec_kernels[1], m->spec_lib, "lstm_spec_kernel_fast"), "cudaLibraryGetKernel");
    check(cudaLibraryGetKernel(&m->lstm_gate_kernels[0], m->spec_lib, "lstm_spec_gates_kernel_exact"), "cudaLibraryGetKernel");
    check(cudaLibraryGetKernel(&m->lstm_gate_kernels[1], m->spec_lib, "lstm_spec_gates_kernel_fast"), "cudaLibraryGetKernel");
    m->spec_state = 1;
    m->spec_note = b.from_cache ? "cubin from cache" : "compiled in " + std::to_string(b.compile_seconds) + " s";
  }
  catch (const CudaError& ex)
  {
    if (m->spec_lib)
      cudaLibraryUnload(m->spec_lib);
    m->spec_lib = nullptr;
    m->spec_state = -1;
    m->spec_note = ex.what();
    if (mode == 1)
      throw;
  }
}

// ---- the general kernel compiled for this model (wavenet_generic_spec.cuh): same policy as the fused family's -------------
void setup_generic_spec_kernel(nam_b200_model* m)
{
  const int mode = jit_mode(m);
  if (!(mode == 1 || ((mode == 0 || mode == 3) && m->opts.max_batch >= 256)) || m->opts.kernel_geometry == 4)
    return;
  SpecBuild b = build_generic_spec_kernel(m->gplan);
  auto give_up = [&](const std::string& why) {
    if (m->spec_lib)
      cudaLibraryUnload(m->spec_lib);
    m->spec_lib = nullptr;
    m->gen_spec_kernel = nullptr;
    m->spec_state = -1;
    m->spec_note = why;
    if (mode == 1)
      throw std::runtime_error("model-specialised kernel unavailable: " + why);
  };
  if (!b.ok)
    return give_up(b.why_not);
  cudaError_t e = cudaLibraryLoadData(&m->spec_lib, b.cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
  if (e == cudaSuccess)
    e = cudaLibraryGetKernel(&m->gen_spec_kernel, m->spec_lib, "wavenet_generic_spec_kernel");
  if (e != cudaSuccess)
  {
    cudaGetLastError();
    return give_up(std::string("loading the specialised general kernel failed: ") + cudaGetErrorString(e));
  }
  m->spec_state = 1;
  m->spec_note = std::string("general kernel, ") + (b.from_cache ? "cubin from cache" : "compiled in " + std::to_string(b.compile_seconds) + " s");
}

void launch_lstm(nam_b200_model* m, const float* d_in, float* d_out, int batch, int n_frames, long in_stride,
                 long out_stride, cudaStream_t st)
{
  if (m->spec_state == 1)
  {
    LstmSpecKernelParams sp{m->d_state, m->state_stride, d_in, d_out, in_stride, out_stride, batch, n_frames};
    void* args[] = {&sp};
    // The step rate is bound by one warp's instruction stream as long as every warp has a scheduler to itself: four
    // lanes per stream (gate-split, 8 streams per warp: a shorter dependent chain per step) while every warp still gets a
    // scheduler of its own (4 x SMs), else one thread per stream (32 per warp: more streams in flight).  kernel_geometry
    // 1 / 2 pins one of them.
    const bool gates = m->spec.lstm.hidden >= 2
                       && (m->opts.kernel_geometry == 1 || (m->opts.kernel_geometry != 2 && (batch + 7) / 8 <= 4 * m->sm_count));
    if (gates)
      CUDA_CHECK(cudaLaunchKernel((const void*)m->lstm_gate_kernels[m->fast_tanh_runtime ? 1 : 0], dim3((batch + 7) / 8), dim3(32),
                                  args, 0, st));
    else
      CUDA_CHECK(cudaLaunchKernel((const void*)m->lstm_spec_kernels[m->fast_tanh_runtime ? 1 : 0], dim3((batch + 31) / 32),
                                  dim3(32), args, 0, st));
    m->launches++;
    return;
  }
  const LstmSpec& ls = m->spec.lstm;
  LstmKernelParams kp{};
  kp.weights = m->d_weights;
  kp.n_weight_floats = (int)m->n_weight_floats;
  kp.state = m->d_state;
  kp.state_stride = (int)m->state_stride;
  kp.in = d_in;
  kp.out = d_out;
  kp.in_stride = in_stride;
  kp.out_stride = out_stride;
  kp.batch = batch;
  kp.n_frames = n_frames;
  kp.num_layers = ls.num_layers;
  kp.input_size = ls.input_size;
  kp.hidden = ls.hidden;
  kp.fast_tanh = m->fast_tanh_runtime;
  kp.in_ch = m->spec.in_channels;
  kp.out_ch = m->spec.out_channels;
  const int H = ls.hidden;
  if (H <= kLstmGroupMaxHidden && ls.num_layers <= kLstmGroupMaxLayers && kp.in_ch == 1 && kp.out_ch == 1)
  {
    // a group of G lanes per stream (lstm_group.cuh)
    const int G = H <= 4 ? 4 : (H <= 8 ? 8 : (H <= 16 ? 16 : 32));
    const int spc = kLstmGroupThreads / G;
    size_t w_floats = 0;
    for (int l = 0; l < ls.num_layers; l++)
    {
      const int W = ((l == 0) ? ls.input_size : H) + H;
      w_floats += (size_t)4 * H * (W | 1) + 4 * H;
    }
    const size_t smem_g = (w_floats + H + 1 + (size_t)2 * spc * (kLstmGroupChunk + 1)) * sizeof(float);
    if (smem_g <= 227 * 1024)
    {
      const int grid_g = (batch + spc - 1) / spc;
      auto launch = [&](auto kern) {
        CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        kern<<<grid_g, kLstmGroupThreads, smem_g, st>>>(kp);
      };
      switch (G)
      {
        case 4: launch(lstm_group_kernel<4>); break;
        case 8: launch(lstm_group_kernel<8>); break;
        case 16: launch(lstm_group_kernel<16>); break;
        default: launch(lstm_group_kernel<32>); break;
      }
      CUDA_CHECK(cudaGetLastError());
      m->launches++;
      return;
    }
  }
  const size_t smem = (((m->n_weight_floats + 3) & ~(size_t)3) + (size_t)ls.num_layers * 2 * H * kLstmThreads
                       + (size_t)4 * H * kLstmThreads + (size_t)2 * kLstmThreads * (kLstmChunk + 1))
                      * sizeof(float);
  ensure_max_dynamic_smem(reinterpret_cast<const void*>(lstm_kernel), m->device, 227 * 1024);
  if (smem > 227 * 1024)
    throw std::runtime_error("LSTM too large for the shared-memory resident kernel");
  const int grid = (batch + kLstmThreads - 1) / kLstmThreads;
  lstm_kernel<<<grid, kLstmThreads, smem, st>>>(kp);
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
}

void launch_linear(nam_b200_model* m, const float* d_in, float* d_out, int batch, int n_frames, long in_stride,
                   long out_stride, cudaStream_t st)
{
  const LinearSpec& li = m->spec.linear;
  LinearKernelParams kp{};
  kp.impulse = m->d_weights;
  kp.rf = li.receptive_field;
  kp.bias = li.bias_value;
  kp.state = m->d_state;
  kp.state_stride = (int)m->state_stride;
  kp.in = d_in;
  kp.out = d_out;
  kp.in_stride = in_stride;
  kp.out_stride = out_stride;
  kp.batch = batch;
  kp.n_frames = n_frames;
  const size_t smem = (((size_t)li.receptive_field + 3) & ~(size_t)3) * 4 + ((size_t)li.receptive_field - 1 + kLinThreads) * 4;
  ensure_max_dynamic_smem(reinterpret_cast<const void*>(linear_kernel), m->device, 227 * 1024);
  if (smem > 227 * 1024)
    throw std::runtime_error("Linear receptive field too long for the direct-form kernel");
  if (batch > 65535)
    throw std::runtime_error("Linear: more than 65535 streams per call (grid.y); split the batch");
  dim3 grid((n_frames + kLinThreads - 1) / kLinThreads, batch);
  linear_kernel<<<grid, kLinThreads, smem, st>>>(kp);
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
  const int hist = li.receptive_field - 1;
  if (hist > 0)
  {
    dim3 g2((hist + 255) / 256, batch);
    linear_update_state_kernel<<<g2, 256, 0, st>>>(kp, m->d_state_tmp);
    CUDA_CHECK(cudaGetLastError());
    m->launches++;
    std::swap(m->d_state, m->d_state_tmp);
  }
}

// Streams per pipelined chunk of a host-buffer call: whole waves of the persistent kernel (4 per chunk), so
// chunking costs no extra tail; 0 = do not chunk (non-WaveNet kernels, general kernel).
int wavenet_chunk_streams(nam_b200_model* m)
{
  if (m->spec.arch != Arch::WaveNet || m->use_generic)
    return 0;
  if (m->spec_state == 1)
    return 4 * m->spec_ctas_per_sm * m->sm_count;
  const int per_sm = m->wn_ctas_per_sm > 0 ? m->wn_ctas_per_sm : (m->wn_geometry == 0 ? 3 : 2);
  return 4 * per_sm * m->sm_count;
}

void launch_convnet(nam_b200_model* m, const float* d_in, float* d_out, int batch, int n_frames, long in_stride,
                    long out_stride, cudaStream_t st)
{
  ConvNetKernelParams kp{};
  kp.weights = m->d_weights;
  kp.net = m->gplan.convnet;
  kp.state = m->d_state;
  kp.state_stride = m->state_stride;
  kp.in = d_in;
  kp.out = d_out;
  kp.in_stride = in_stride;
  kp.out_stride = out_stride;
  kp.batch = batch;
  kp.n_frames = n_frames;
  kp.t_base = m->t_base;
  kp.n_weight_floats = (int)((m->n_weight_floats + 3) & ~(size_t)3);
  const size_t wbytes = (size_t)kp.n_weight_floats * sizeof(float);
  const int grid = std::min(batch, 16 * m->sm_count);
  if (wbytes <= 200 * 1024)
  {
    ensure_max_dynamic_smem(reinterpret_cast<const void*>(convnet_kernel<true>), m->device, 200 * 1024);
    convnet_kernel<true><<<grid, kGenTile, wbytes, st>>>(kp);
  }
  else
    convnet_kernel<false><<<grid, kGenTile, 0, st>>>(kp);
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
}

// Run the hot path on device buffers and advance the stream clock.
void run_device(nam_b200_model* m, const float* d_in, float* d_out, int batch, int n_frames, long in_stride,
                long out_stride, cudaStream_t st)
{
  switch (m->spec.arch)
  {
    case Arch::WaveNet: launch_wavenet(m, d_in, d_out, batch, n_frames, in_stride, out_stride, st); break;
    case Arch::LSTM: launch_lstm(m, d_in, d_out, batch, n_frames, in_stride, out_stride, st); break;
    case Arch::Linear: launch_linear(m, d_in, d_out, batch, n_frames, in_stride, out_stride, st); break;
    case Arch::ConvNet: launch_convnet(m, d_in, d_out, batch, n_frames, in_stride, out_stride, st); break;
    default: throw std::runtime_error("no kernel for this architecture");
  }
  m->t_base += (uint32_t)n_frames;
  m->streams_identical = false; // (prewarm() restores the flag: it feeds every stream the same zeros)
}

void ensure_staging(nam_b200_model* m, size_t floats)
{
  if (floats <= m->staging_floats)
    return;
  if (m->d_in)
    cudaFree(m->d_in);
  if (m->d_out)
    cudaFree(m->d_out);
  m->d_in = m->d_out = nullptr;
  m->staging_floats = 0;
  CUDA_CHECK(cudaMalloc(&m->d_in, floats * sizeof(float)));
  CUDA_CHECK(cudaMalloc(&m->d_out, floats * sizeof(float)));
  m->staging_floats = floats;
}

void ensure_pinned(nam_b200_model* m, size_t floats)
{
  if (floats <= m->h_pin_floats)
    return;
  if (m->h_pin)
    cudaFreeHost(m->h_pin);
  m->h_pin = m->h_pin_dev = nullptr;
  m->h_pin_floats = 0;
  CUDA_CHECK(cudaHostAlloc(&m->h_pin, floats * sizeof(float), cudaHostAllocMapped));
  m->h_pin_floats = floats;
  if (cudaHostGetDevicePointer(&m->h_pin_dev, m->h_pin, 0) != cudaSuccess)
  {
    cudaGetLastError();
    m->h_pin_dev = nullptr; // no zero-copy on this device: the planar calls fall back to explicit copies
  }
}

// Zero the state, set the trained initial state where the architecture has one.
void init_state(nam_b200_model* m)
{
  const size_t total = (size_t)m->state_stride * m->opts.max_batch;
  CUDA_CHECK(cudaMemsetAsync(m->d_state, 0, total * sizeof(float), m->stream));
  if (m->spec.arch == Arch::LSTM)
  {
    // h0 / c0 are trained parameters (lstm.cpp:24-28): stream 0 gets them, then broadcast
    std::vector<float> st((size_t)m->state_stride, 0.0f);
    const int H = m->spec.lstm.hidden;
    for (int l = 0; l < m->spec.lstm.num_layers; l++)
    {
      std::copy(m->spec.lstm.cells[l].h0.begin(), m->spec.lstm.cells[l].h0.end(), st.begin() + (size_t)l * 2 * H);
      std::copy(m->spec.lstm.cells[l].c0.begin(), m->spec.lstm.cells[l].c0.end(), st.begin() + (size_t)l * 2 * H + H);
    }
    CUDA_CHECK(cudaMemcpyAsync(m->d_state, st.data(), st.size() * sizeof(float), cudaMemcpyHostToDevice, m->stream));
    CUDA_CHECK(cudaStreamSynchronize(m->stream));
  }
  if (m->spec.arch == Arch::Linear && m->d_state_tmp)
    CUDA_CHECK(cudaMemsetAsync(m->d_state_tmp, 0, total * sizeof(float), m->stream));
  m->t_base = 0;
  m->streams_identical = true;
  m->state_initialised = true;
}

void broadcast_state(nam_b200_model* m)
{
  const int batch = m->opts.max_batch;
  if (batch <= 1 || m->state_stride == 0)
    return;
  dim3 grid((unsigned)std::min<long>((m->state_stride / 4 + 255) / 256, 1024), (unsigned)std::min(batch - 1, 64));
  if (grid.x < 1)
    grid.x = 1;
  broadcast_state_kernel<<<grid, 256, 0, m->stream>>>(m->d_state, m->state_stride, batch);
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
}

// DSP::prewarm (dsp.cpp:67-101): zeros in max_frames blocks until >= prewarm_samples; done once on
// stream 0 (every stream would compute the identical state) and broadcast.
void prewarm(nam_b200_model* m)
{
  const int ps = m->spec.prewarm_samples;
  if (ps <= 0)
    return;
  const int bs = std::max(m->max_frames, 1);
  const size_t ci = (size_t)m->spec.in_channels, co = (size_t)m->spec.out_channels;
  ensure_staging(m, (size_t)m->opts.max_batch * bs * std::max(ci, co));
  // DSP::prewarm continues from the instance's CURRENT state (dsp.cpp:67-101).  Straight after init_state every stream
  // would compute the same thing: stream 0 runs, its state is broadcast.  Once the streams have seen different audio
  // (a standalone nam_b200_prewarm, or a Reset of an LSTM, which keeps its running state) all of them are prewarmed.
  const int nb = m->streams_identical ? 1 : m->opts.max_batch;
  CUDA_CHECK(cudaMemsetAsync(m->d_in, 0, (size_t)nb * bs * ci * sizeof(float), m->stream));
  const bool identical = m->streams_identical;
  int done = 0;
  while (done < ps)
  {
    run_device(m, m->d_in, m->d_out, nb, bs, (long)(bs * ci), (long)(bs * co), m->stream);
    done += bs;
  }
  m->streams_identical = identical; // zeros into identical streams keep them identical
  if (identical)
    broadcast_state(m);
  if (m->spec.arch == Arch::Linear && m->d_state_tmp)
    CUDA_CHECK(cudaMemcpyAsync(m->d_state_tmp, m->d_state, (size_t)m->state_stride * m->opts.max_batch * sizeof(float),
                               cudaMemcpyDeviceToDevice, m->stream));
  CUDA_CHECK(cudaStreamSynchronize(m->stream));
}

int create_common(ModelSpec&& spec, const nam_b200_options* user_opts, nam_b200_model** out)
{
  std::unique_ptr<nam_b200_model> m(new nam_b200_model());
  nam_b200_default_options(&m->opts);
  if (user_opts)
  {
    const size_t n = std::min<size_t>(sizeof(nam_b200_options), (size_t)std::max(user_opts->struct_size, 0));
    std::memcpy(&m->opts, user_opts, n);
    m->opts.struct_size = sizeof(nam_b200_options);
  }
  if (m->opts.max_batch < 1)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "max_batch must be >= 1");
  m->spec = std::move(spec);
  m->fast_tanh_runtime = m->opts.fast_tanh;
  if (const char* e = std::getenv("NAM_B200_TIMING"))
    m->opts_timing_events = (*e == '1');

  if (m->spec.arch == Arch::Container)
  {
    // ContainerConfig::create (container.cpp:146-169): every sub-model goes through get_dsp() on its own
    LoadOptions lo;
    lo.fast_tanh = m->opts.fast_tanh != 0;
    for (const auto& sub : m->spec.submodels)
    {
      nam_b200_model* h = nullptr;
      int rc;
      try
      {
        rc = create_common(model_spec_from_text(sub.model_json, lo), &m->opts, &h);
      }
      catch (const std::exception& ex)
      {
        return fail(NAM_B200_ERR_MODEL, ex.what());
      }
      if (rc != NAM_B200_OK)
        return rc;
      m->subs.emplace_back(h);
      // container.cpp:35-46
      const double sr = h->spec.sample_rate, want = m->spec.sample_rate;
      if (sr != want && sr != -1.0 && want != -1.0)
        return fail(NAM_B200_ERR_MODEL, "ContainerModel: submodel sample rate mismatch (expected " + std::to_string(want)
                                          + ", got " + std::to_string(sr) + ")");
    }
    m->active_sub = (int)m->subs.size() - 1; // default to full size (container.cpp:49)
    m->device = m->subs.back()->device;
    *out = m.release();
    return NAM_B200_OK;
  }

  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(NAM_B200_ERR_CUDA, std::string("no usable CUDA device (libnam_b200 has no CPU path): ")
                                     + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"));
  try
  {
    if (m->opts.device >= 0)
      CUDA_CHECK(cudaSetDevice(m->opts.device));
    CUDA_CHECK(cudaGetDevice(&m->device));
    cudaDeviceProp prop{};
    CUDA_CHECK(cudaGetDeviceProperties(&prop, m->device));
    m->sm_count = prop.multiProcessorCount;
    CUDA_CHECK(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
    CUDA_CHECK(cudaEventCreate(&m->ev0));
    CUDA_CHECK(cudaEventCreate(&m->ev1));

    // multi-channel models: WaveNet through the general kernel, LSTM through the thread-per-stream kernel
    const bool mono = m->spec.in_channels == 1 && m->spec.out_channels == 1;
    if (!mono && m->spec.arch == Arch::Linear)
      return fail(NAM_B200_ERR_UNSUPPORTED, "Linear on the CUDA path is mono in / mono out (model has "
                                              + std::to_string(m->spec.in_channels) + " in, "
                                              + std::to_string(m->spec.out_channels) + " out channels)");
    std::vector<float> blob;
    switch (m->spec.arch)
    {
      case Arch::WaveNet:
      {
        m->plan = plan_wavenet(m->spec);
        if (!mono && m->plan.eligible)
        {
          m->plan.eligible = false;
          m->plan.why_not = "multi-channel in / out";
        }
        if (m->plan.eligible && m->opts.kernel_geometry != 3
            && wavenet_smem_bytes(m->plan, m->opts.kernel_geometry == 1 ? 0 : 1) > 227 * 1024)
        {
          // e.g. > ~50 layers of 16 channels: the general kernel keeps such weights in global memory
          m->plan.eligible = false;
          m->plan.why_not = "packed weights + tile exceed the 227 KB of shared memory of the fused kernel";
        }
        if (!m->plan.eligible || m->opts.kernel_geometry == 4)
        {
          // outside the fused families (or asked for explicitly): the general kernel
          m->gplan = plan_generic(m->spec);
          if (!m->gplan.eligible)
            return fail(NAM_B200_ERR_UNSUPPORTED,
                        "WaveNet not supported on the CUDA path: fused kernel: "
                          + (m->plan.eligible ? std::string("(eligible)") : m->plan.why_not) + "; general kernel: " + m->gplan.why_not);
          m->use_generic = true;
          setup_generic_spec_kernel(m.get()); // throws when jit = 1 and the specialised general kernel cannot be had
          blob = m->gplan.weights;
          m->state_stride = m->gplan.state_floats;
          m->flops_per_frame = 2.0 * m->gplan.macs_per_frame;
          m->variant = 9000;
          CUDA_CHECK(cudaMalloc(&m->d_glayers, std::max<size_t>(m->gplan.layers.size(), 1) * sizeof(GLayer)));
          CUDA_CHECK(cudaMemcpy(m->d_glayers, m->gplan.layers.data(), m->gplan.layers.size() * sizeof(GLayer),
                                cudaMemcpyHostToDevice));
          break;
        }
        blob = m->plan.blob;
        m->state_stride = m->plan.state_floats;
        m->flops_per_frame = 2.0 * m->plan.macs_per_frame;
        m->variant = m->plan.cp[0] * 100 + (m->plan.n_arrays > 1 ? m->plan.cp[1] : 0);
        // option: 0 default, 1 = FFMA 128-thread, 2 = FFMA 256-thread, 3 = tensor-core (none on sm_90a)
        if (m->opts.kernel_geometry == 3)
          return fail(NAM_B200_ERR_UNSUPPORTED, "tensor-core WaveNet kernel: this sm_90a library has none (use kernel_geometry "
                                                "0, 1, 2 or 4)");
        m->wn_geometry = (m->opts.kernel_geometry == 1) ? 0 : 1;
        if (wavenet_smem_bytes(m->plan, m->wn_geometry) > 227 * 1024)
          return fail(NAM_B200_ERR_UNSUPPORTED, "WaveNet weights do not fit in shared memory");
        setup_spec_kernel(m.get());
        break;
      }
      case Arch::LSTM:
      {
        const LstmSpec& ls = m->spec.lstm;
        if (ls.input_size != m->spec.in_channels) // lstm.cpp:74,111: in_channels samples land in an input_size vector
          return fail(NAM_B200_ERR_UNSUPPORTED, "LSTM input_size (" + std::to_string(ls.input_size) + ") != in_channels ("
                                                  + std::to_string(m->spec.in_channels) + ")");
        if ((int)ls.head_b.size() != m->spec.out_channels || m->spec.out_channels > 64)
          return fail(NAM_B200_ERR_UNSUPPORTED, "LSTM head with " + std::to_string(ls.head_b.size()) + " rows for "
                                                  + std::to_string(m->spec.out_channels) + " output channels");
        if (ls.num_layers < 1)
          return fail(NAM_B200_ERR_UNSUPPORTED, "LSTM with zero layers");
        double macs = 0.0;
        for (const auto& c : ls.cells)
        {
          blob.insert(blob.end(), c.w.begin(), c.w.end());
          blob.insert(blob.end(), c.b.begin(), c.b.end());
          macs += 4.0 * c.hidden * (c.input_size + c.hidden);
        }
        blob.insert(blob.end(), ls.head_w.begin(), ls.head_w.end());
        blob.insert(blob.end(), ls.head_b.begin(), ls.head_b.end());
        macs += (double)ls.hidden * m->spec.out_channels;
        m->state_stride = ((long)ls.num_layers * 2 * ls.hidden + 3) & ~3L;
        m->flops_per_frame = 2.0 * macs;
        m->variant = 2000 + ls.hidden;
        setup_lstm_spec_kernel(m.get());
        break;
      }
      case Arch::Linear:
      {
        blob = m->spec.linear.impulse;
        m->state_stride = ((long)std::max(m->spec.linear.receptive_field - 1, 1) + 3) & ~3L;
        m->flops_per_frame = 2.0 * m->spec.linear.receptive_field;
        m->variant = 3000;
        break;
      }
      case Arch::ConvNet:
      {
        m->gplan = plan_convnet(m->spec);
        if (!m->gplan.eligible)
          return fail(NAM_B200_ERR_UNSUPPORTED, "ConvNet not supported on the CUDA path: " + m->gplan.why_not);
        blob = m->gplan.weights;
        m->state_stride = std::max(m->gplan.state_floats, 4L);
        m->flops_per_frame = 2.0 * m->gplan.macs_per_frame;
        m->variant = 9500;
        break;
      }
      default: return fail(NAM_B200_ERR_UNSUPPORTED, "no CUDA kernel for architecture " + m->spec.architecture);
    }
    m->n_weight_floats = blob.size();
    const size_t alloc_floats = (blob.size() + 3) & ~(size_t)3;
    blob.resize(alloc_floats, 0.0f);
    CUDA_CHECK(cudaMalloc(&m->d_weights, alloc_floats * sizeof(float)));
    CUDA_CHECK(cudaMemcpy(m->d_weights, blob.data(), alloc_floats * sizeof(float), cudaMemcpyHostToDevice));
    const size_t state_total = (size_t)m->state_stride * m->opts.max_batch;
    CUDA_CHECK(cudaMalloc(&m->d_state, std::max<size_t>(state_total, 4) * sizeof(float)));
    if (m->spec.arch == Arch::Linear)
      CUDA_CHECK(cudaMalloc(&m->d_state_tmp, std::max<size_t>(state_total, 4) * sizeof(float)));
    init_state(m.get());
    CUDA_CHECK(cudaStreamSynchronize(m->stream));
  }
  catch (const CudaError& ex)
  {
    return fail(NAM_B200_ERR_CUDA, ex.what());
  }
  catch (const std::exception& ex)
  {
    return fail(NAM_B200_ERR_MODEL, ex.what());
  }
  *out = m.release();
  return NAM_B200_OK;
}

template <typename F>
int guarded(nam_b200_model* m, F&& body)
{
  if (!m)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null model handle");
  try
  {
    CUDA_CHECK(cudaSetDevice(m->device));
    return body();
  }
  catch (const CudaError& ex)
  {
    return fail(NAM_B200_ERR_CUDA, ex.what());
  }
  catch (const std::exception& ex)
  {
    return fail(NAM_B200_ERR_MODEL, ex.what());
  }
}

int check_process_args(nam_b200_model* m, const void* in, const void* out, int batch, int n_frames)
{
  if (!in || !out)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null audio buffer");
  if (!m->is_reset)
    return fail(NAM_B200_ERR_STATE, "process called before reset");
  if (batch < 1 || batch > m->opts.max_batch)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT,
                "batch " + std::to_string(batch) + " outside [1, max_batch=" + std::to_string(m->opts.max_batch) + "]");
  if (n_frames < 0 || n_frames > m->max_frames)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "n_frames " + std::to_string(n_frames) + " exceeds max_frames "
                                                 + std::to_string(m->max_frames) + " of the last reset");
  return NAM_B200_OK;
}

// SlimmableContainer handles forward to their active sub-model (ContainerModel::process etc., container.cpp:52-63)
nam_b200_model* active_model(nam_b200_model* m)
{
  return (m && m->active_sub >= 0) ? m->subs[(size_t)m->active_sub].get() : m;
}
const nam_b200_model* active_model(const nam_b200_model* m)
{
  return (m && m->active_sub >= 0) ? m->subs[(size_t)m->active_sub].get() : m;
}

// nam::DSP::process for stream 0: the caller's channel arrays go through the handle's pinned scratch (double -> float
// is the cast of model.cpp:817 / lstm.cpp:111).  Small calls -- the plugin protocol: one stream, 64..1024 frames --
// skip both copies: the scratch is mapped into the device's address space, the kernel reads its input from it and
// writes its output to it directly (two DMA round trips less per call; the reference's benchmodel spends most of a
// 64-frame call on latency, not on arithmetic).
constexpr size_t kZeroCopyFloats = 8192;

template <typename T>
int process_planar(nam_b200_model* m, const T* const* input, T* const* output, int n_frames)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    if (!input || !output)
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null channel array");
    const int rc = check_process_args(m, input[0], output[0], 1, n_frames);
    if (rc != NAM_B200_OK)
      return rc;
    if (n_frames == 0)
      return NAM_B200_OK;
    const size_t ci = (size_t)m->spec.in_channels, co = (size_t)m->spec.out_channels, n = (size_t)n_frames;
    float* hin = m->h_pin;
    float* hout = m->h_pin + (size_t)m->max_frames * std::max(ci, co);
    for (size_t c = 0; c < ci; c++)
      for (size_t i = 0; i < n; i++)
        hin[c * n + i] = (float)input[c][i];
    if ((ci + co) * n <= kZeroCopyFloats && m->h_pin_dev != nullptr)
    {
      float* din = m->h_pin_dev;
      float* dout = m->h_pin_dev + (hout - hin);
      m->flag_pending = false;
      const bool doorbell = m->h_flag_dev != nullptr && n_frames <= 128 && !m->opts_timing_events;
      if (!doorbell)
        CUDA_CHECK(cudaEventRecord(m->ev0, m->stream));
      run_device(m, din, dout, 1, n_frames, (long)(ci * n), (long)(co * n), m->stream);
      if (doorbell && m->flag_pending)
      {
        // the low-latency kernel served the call: wait for its doorbell (a word of host memory) -- no stream
        // synchronisation, no event records on the per-block path
        const unsigned want = m->flag_seq;
        volatile unsigned* flag = m->h_flag;
        long spins = 0;
        while (*flag != want)
          if (++spins > (1L << 26))
          {
            CUDA_CHECK(cudaStreamSynchronize(m->stream)); // surfaces a launch / execution error instead of hanging
            break;
          }
        m->timing_valid = false;
        for (size_t c = 0; c < co; c++)
          for (size_t i = 0; i < n; i++)
            output[c][i] = (T)hout[c * n + i];
        return NAM_B200_OK;
      }
      CUDA_CHECK(cudaEventRecord(m->ev1, m->stream));
    }
    else
    {
      CUDA_CHECK(cudaMemcpyAsync(m->d_in, hin, ci * n * sizeof(float), cudaMemcpyHostToDevice, m->stream));
      CUDA_CHECK(cudaEventRecord(m->ev0, m->stream));
      run_device(m, m->d_in, m->d_out, 1, n_frames, (long)(ci * n), (long)(co * n), m->stream);
      CUDA_CHECK(cudaEventRecord(m->ev1, m->stream));
      CUDA_CHECK(cudaMemcpyAsync(hout, m->d_out, co * n * sizeof(float), cudaMemcpyDeviceToHost, m->stream));
    }
    CUDA_CHECK(cudaStreamSynchronize(m->stream));
    m->timing_valid = true;
    for (size_t c = 0; c < co; c++)
      for (size_t i = 0; i < n; i++)
        output[c][i] = (T)hout[c * n + i];
    return NAM_B200_OK;
  });
}

} // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

void nam_b200_default_options(nam_b200_options* opts)
{
  if (!opts)
    return;
  std::memset(opts, 0, sizeof(*opts));
  opts->struct_size = sizeof(nam_b200_options);
  opts->device = -1;
  opts->max_batch = 1;
  opts->fast_tanh = 0;
  opts->prewarm_on_reset = 1;
  opts->ctas_per_sm = 0;
}

int nam_b200_abi_version(void)
{
  return NAM_B200_ABI_VERSION;
}

const char* nam_b200_last_error(void)
{
  return g_last_error.c_str();
}

int nam_b200_create_from_file(const char* nam_path, const nam_b200_options* opts, nam_b200_model** out)
{
  if (!nam_path || !out)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  LoadOptions lo;
  lo.fast_tanh = opts ? (opts->fast_tanh != 0) : false;
  try
  {
    ModelSpec spec = model_spec_from_file(nam_path, lo);
    return create_common(std::move(spec), opts, out);
  }
  catch (const NamFileValidationError& ex)
  {
    return fail(NAM_B200_ERR_FILE, ex.what());
  }
  catch (const std::exception& ex)
  {
    return fail(NAM_B200_ERR_MODEL, ex.what());
  }
}

int nam_b200_create_from_json(const char* nam_json_text, const nam_b200_options* opts, nam_b200_model** out)
{
  if (!nam_json_text || !out)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  LoadOptions lo;
  lo.fast_tanh = opts ? (opts->fast_tanh != 0) : false;
  try
  {
    ModelSpec spec = model_spec_from_text(nam_json_text, lo);
    return create_common(std::move(spec), opts, out);
  }
  catch (const json::ParseError& ex)
  {
    return fail(NAM_B200_ERR_FILE, ex.what());
  }
  catch (const std::exception& ex)
  {
    return fail(NAM_B200_ERR_MODEL, ex.what());
  }
}

void nam_b200_destroy(nam_b200_model* m)
{
  delete m;
}

static int inspect_spec(const ModelSpec& spec, char* out, int64_t capacity)
{
  if (!out || capacity <= 0)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null output buffer");
  std::string kernel = "unsupported", reason;
  double flops = 0.0;
  long state_floats = 0;
  int variant = 0;
  if (spec.arch == Arch::Container)
  {
    // describe the default (largest) sub-model; the container itself only dispatches
    LoadOptions lo;
    const int rc = inspect_spec(model_spec_from_text(spec.submodels.back().model_json, lo), out, capacity);
    if (rc != NAM_B200_OK)
      return rc;
    std::string text(out);
    const std::string tag = "{\"architecture\": \"";
    if (text.compare(0, tag.size(), tag) == 0)
      text = "{\"container\": \"SlimmableContainer\", \"submodels\": " + std::to_string(spec.submodels.size())
             + ", \"architecture\": \"" + text.substr(tag.size());
    std::snprintf(out, (size_t)capacity, "%s", text.c_str());
    return NAM_B200_OK;
  }
  const bool mono = spec.in_channels == 1 && spec.out_channels == 1;
  if (!mono && spec.arch == Arch::Linear)
    reason = "Linear on the CUDA path is mono in / mono out";
  else if (spec.arch == Arch::WaveNet)
  {
    WaveNetPlan plan = plan_wavenet(spec);
    if (!mono && plan.eligible)
    {
      plan.eligible = false;
      plan.why_not = "multi-channel in / out";
    }
    if (plan.eligible)
    {
      kernel = "fused";
      flops = 2.0 * plan.macs_per_frame;
      state_floats = plan.state_floats;
      variant = plan.cp[0] * 100 + (plan.n_arrays > 1 ? plan.cp[1] : 0);
    }
    else
    {
      const GenericPlan gp = plan_generic(spec);
      if (gp.eligible)
      {
        kernel = "generic";
        flops = 2.0 * gp.macs_per_frame;
        state_floats = gp.state_floats;
        variant = 9000;
        reason = "fused kernel: " + plan.why_not;
      }
      else
        reason = plan.why_not + "; general kernel: " + gp.why_not;
    }
  }
  else if (spec.arch == Arch::LSTM)
  {
    if (spec.lstm.input_size != spec.in_channels || spec.lstm.num_layers < 1)
      reason = "LSTM input_size != in_channels or no layers";
    else
    {
      kernel = "lstm";
      double macs = (double)spec.lstm.hidden * spec.out_channels;
      for (const auto& c : spec.lstm.cells)
        macs += 4.0 * c.hidden * (c.input_size + c.hidden);
      flops = 2.0 * macs;
      state_floats = (long)spec.lstm.num_layers * 2 * spec.lstm.hidden;
      variant = 2000 + spec.lstm.hidden;
    }
  }
  else if (spec.arch == Arch::ConvNet)
  {
    const GenericPlan gp = plan_convnet(spec);
    if (gp.eligible)
    {
      kernel = "convnet";
      flops = 2.0 * gp.macs_per_frame;
      state_floats = gp.state_floats;
      variant = 9500;
    }
    else
      reason = gp.why_not;
  }
  else
  {
    kernel = "linear";
    flops = 2.0 * spec.linear.receptive_field;
    state_floats = std::max(spec.linear.receptive_field - 1, 0);
    variant = 3000;
  }
  for (auto& ch : reason)
    if (ch == '"' || ch == '\\' || ch == '\n')
      ch = ' ';
  char buf[1024];
  std::snprintf(buf, sizeof(buf),
                "{\"architecture\": \"%s\", \"in_channels\": %d, \"out_channels\": %d, \"prewarm_samples\": %d, "
                "\"n_weights\": %zu, \"expected_sample_rate\": %.17g, \"flops_per_frame\": %.17g, "
                "\"state_bytes_per_stream\": %ld, \"kernel\": \"%s\", \"kernel_variant\": %d, \"has_loudness\": %s, "
                "\"loudness\": %.17g, \"reason\": \"%s\"}",
                spec.architecture.c_str(), spec.in_channels, spec.out_channels, spec.prewarm_samples, spec.n_weights,
                spec.sample_rate, flops, state_floats * 4, kernel.c_str(), variant, spec.loudness ? "true" : "false",
                spec.loudness.value_or(0.0), reason.c_str());
  std::snprintf(out, (size_t)capacity, "%s", buf);
  return NAM_B200_OK;
}

int nam_b200_inspect_json(const char* nam_json_text, int fast_tanh, char* out, int64_t capacity)
{
  if (!nam_json_text)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument");
  LoadOptions lo;
  lo.fast_tanh = fast_tanh != 0;
  try
  {
    return inspect_spec(model_spec_from_text(nam_json_text, lo), out, capacity);
  }
  catch (const json::ParseError& ex)
  {
    return fail(NAM_B200_ERR_FILE, ex.what());
  }
  catch (const std::exception& ex)
  {
    return fail(NAM_B200_ERR_MODEL, ex.what());
  }
}

int nam_b200_jit_prepare_json(const char* nam_json_text, int fast_tanh, char* out, int64_t capacity)
{
  return nam_b200_jit_prepare_json_for_batch(nam_json_text, fast_tanh, 1, out, capacity);
}

int nam_b200_jit_prepare_json_for_batch(const char* nam_json_text, int fast_tanh, int max_batch, char* out, int64_t capacity)
{
  if (!nam_json_text)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument");
  LoadOptions lo;
  lo.fast_tanh = fast_tanh != 0;
  try
  {
    const ModelSpec ms = model_spec_from_text(nam_json_text, lo);
    if (ms.arch != Arch::WaveNet && ms.arch != Arch::LSTM)
      return fail(NAM_B200_ERR_UNSUPPORTED, "only WaveNets and LSTMs have model-specialised kernels");
    SpecBuild b;
    bool fused_family = false;
    if (ms.arch == Arch::LSTM)
      b = build_lstm_spec_kernel(ms);
    else
    {
      const WaveNetPlan wp = plan_wavenet(ms);
      fused_family = wp.eligible && ms.in_channels == 1 && ms.out_channels == 1;
      b = fused_family ? build_spec_kernel(wp, spec_geometry_for(std::max(max_batch, 1), 132))  // H100 SXM
                       : build_generic_spec_kernel(plan_generic(ms)); // every other WaveNet: the general kernel, compiled
    }
    // WaveNets: also the low-latency kernel for 64-frame calls (the plugin protocol), so that a first Reset finds it cached
    SpecBuild lat;
    if (ms.arch == Arch::WaveNet && fused_family)
      lat = build_lat_kernel(plan_wavenet(ms), 2);
    std::string why;
    for (char c : b.why_not.substr(0, 600))
      why += (c == '"' || c == '\\') ? '\'' : (c == '\n' ? ' ' : c);
    char buf[1024];
    std::snprintf(buf, sizeof buf,
                  "{\"ok\": %s, \"from_cache\": %s, \"compile_seconds\": %.3f, \"cubin_bytes\": %zu, \"threads\": %d, "
                  "\"frames_per_thread\": %d, \"smem_bytes\": %zu, \"why_not\": \"%s\", \"lat_ok\": %s, "
                  "\"lat_compile_seconds\": %.3f, \"lat_cubin_bytes\": %zu}",
                  b.ok ? "true" : "false", b.from_cache ? "true" : "false", b.compile_seconds, b.cubin.size() + b.cubin_extra.size(), b.geom.nt,
                  b.geom.s, b.ok ? b.smem_bytes() : (size_t)0, why.c_str(), lat.ok ? "true" : "false", lat.compile_seconds,
                  lat.cubin.size());
    if (out && capacity > 0)
    {
      std::strncpy(out, buf, (size_t)capacity - 1);
      out[capacity - 1] = '\0';
    }
    return NAM_B200_OK;
  }
  catch (const json::ParseError& ex)
  {
    return fail(NAM_B200_ERR_FILE, ex.what());
  }
  catch (const std::exception& ex)
  {
    return fail(NAM_B200_ERR_MODEL, ex.what());
  }
}

int64_t nam_b200_jit_note(const nam_b200_model* m, char* out, int64_t capacity)
{
  m = active_model(m);
  if (!m)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null model handle");
  const std::string note = m->spec_note + (m->lat_note.empty() ? "" : (m->spec_note.empty() ? "" : "; ") + ("low-latency kernel: " + m->lat_note));
  if (out && capacity > 0)
  {
    std::strncpy(out, note.c_str(), (size_t)capacity - 1);
    out[capacity - 1] = '\0';
  }
  return (int64_t)note.size();
}

int nam_b200_inspect_file(const char* nam_path, int fast_tanh, char* out, int64_t capacity)
{
  if (!nam_path)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument");
  LoadOptions lo;
  lo.fast_tanh = fast_tanh != 0;
  try
  {
    return inspect_spec(model_spec_from_file(nam_path, lo), out, capacity);
  }
  catch (const NamFileValidationError& ex)
  {
    return fail(NAM_B200_ERR_FILE, ex.what());
  }
  catch (const std::exception& ex)
  {
    return fail(NAM_B200_ERR_MODEL, ex.what());
  }
}

int64_t nam_b200_submodel_json(const char* nam_json_text, int index, double* max_value, char* out, int64_t capacity)
{
  if (!nam_json_text)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument");
  try
  {
    LoadOptions lo;
    const ModelSpec spec = model_spec_from_text(nam_json_text, lo);
    if (spec.arch != Arch::Container)
      return index < 0 ? 0 : fail(NAM_B200_ERR_UNSUPPORTED, "model is not slimmable");
    if (index < 0)
      return (int64_t)spec.submodels.size();
    if ((size_t)index >= spec.submodels.size())
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, "sub-model index out of range");
    const ModelSpec::Submodel& sm = spec.submodels[(size_t)index];
    if (max_value)
      *max_value = sm.max_value;
    if (out && capacity > 0)
    {
      const size_t n = std::min((size_t)capacity - 1, sm.model_json.size());
      std::memcpy(out, sm.model_json.data(), n);
      out[n] = 0;
    }
    return (int64_t)sm.model_json.size();
  }
  catch (const std::exception& ex)
  {
    return fail(NAM_B200_ERR_MODEL, ex.what());
  }
}

int nam_b200_get_info(const nam_b200_model* m, nam_b200_info* info)
{
  m = active_model(m);
  if (!m || !info)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument");
  nam_b200_info r;
  std::memset(&r, 0, sizeof(r));
  r.struct_size = sizeof(nam_b200_info);
  r.architecture = (int)m->spec.arch;
  r.in_channels = m->spec.in_channels;
  r.out_channels = m->spec.out_channels;
  r.prewarm_samples = m->spec.prewarm_samples;
  r.max_batch = m->opts.max_batch;
  r.max_frames = m->max_frames;
  r.has_loudness = m->spec.loudness.has_value();
  r.has_input_level = m->spec.input_level.has_value();
  r.has_output_level = m->spec.output_level.has_value();
  r.expected_sample_rate = m->spec.sample_rate;
  r.loudness = m->spec.loudness.value_or(0.0);
  r.input_level_dbu = m->spec.input_level.value_or(0.0);
  r.output_level_dbu = m->spec.output_level.value_or(0.0);
  r.n_weights = (int64_t)m->spec.n_weights;
  r.state_bytes_per_stream = (int64_t)m->state_stride * 4;
  r.flops_per_frame = m->flops_per_frame;
  r.kernel_variant = m->variant;
  r.jit_state = m->spec_state;
  r.jit_lat_state = m->lat_state;
  const size_t n = std::min<size_t>(sizeof(r), (size_t)std::max(info->struct_size, 0));
  const int32_t user_size = info->struct_size;
  std::memcpy(info, &r, n);
  info->struct_size = user_size;
  return NAM_B200_OK;
}

int nam_b200_reset(nam_b200_model* m, double sample_rate, int max_frames)
{
  // like the reference, the external rate is recorded but does not change the arithmetic
  if (m && m->active_sub >= 0)
  {
    // ContainerModel::Reset (container.cpp:73-86): remember the settings, reset only the active sub-model
    if (max_frames < 1)
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, "max_frames must be >= 1");
    m->ext_sample_rate = sample_rate;
    m->max_frames = max_frames;
    m->is_reset = true;
    m = active_model(m);
  }
  return guarded(m, [&]() -> int {
    if (max_frames < 1)
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, "max_frames must be >= 1");
    m->max_frames = max_frames;
    const size_t ch = (size_t)std::max(m->spec.in_channels, m->spec.out_channels);
    ensure_staging(m, (size_t)m->opts.max_batch * max_frames * ch);
    ensure_pinned(m, (size_t)2 * max_frames * ch);
    ensure_hist(m);
    setup_lat_kernel(m);
    if (m->spec.arch == Arch::WaveNet && !m->h_flag && m->opts.max_batch <= m->sm_count && max_frames <= 128
        && cudaHostAlloc(&m->h_flag, 64, cudaHostAllocMapped) == cudaSuccess)
    {
      // completion doorbell of the low-latency kernels: DSP::process spins on this word instead of synchronising
      *m->h_flag = 0;
      if (cudaHostGetDevicePointer(&m->h_flag_dev, m->h_flag, 0) != cudaSuccess)
        m->h_flag_dev = nullptr;
    }
    cudaGetLastError();
    // DSP::Reset = SetMaxBufferSize + prewarm (dsp.cpp:130-140).  WaveNet / ConvNet / Linear clear their buffers in
    // SetMaxBufferSize (RingBuffer::Reset, Buffer::_reset_input_buffer); the reference's LSTM overrides neither, so its
    // hidden and cell state SURVIVE a Reset and only the prewarm runs on top of it: a second Reset keeps the state here too.
    if (!(m->spec.arch == Arch::LSTM && m->state_initialised))
      init_state(m);
    m->is_reset = true;
    CUDA_CHECK(cudaEventRecord(m->ev0, m->stream));
    if (m->opts.prewarm_on_reset)
      prewarm(m);
    CUDA_CHECK(cudaEventRecord(m->ev1, m->stream));
    CUDA_CHECK(cudaStreamSynchronize(m->stream));
    m->timing_valid = true;
    return NAM_B200_OK;
  });
}

int nam_b200_prewarm(nam_b200_model* m)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    if (!m->is_reset)
      return fail(NAM_B200_ERR_STATE, "prewarm called before reset");
    prewarm(m);
    return NAM_B200_OK;
  });
}

int nam_b200_process_f32_device(nam_b200_model* m, const float* in_device, float* out_device, int batch, int n_frames,
                                int64_t in_stride, int64_t out_stride, void* cuda_stream)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    const int rc = check_process_args(m, in_device, out_device, batch, n_frames);
    if (rc != NAM_B200_OK)
      return rc;
    if (n_frames == 0)
      return NAM_B200_OK;
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : m->stream;
    CUDA_CHECK(cudaEventRecord(m->ev0, st));
    run_device(m, in_device, out_device, batch, n_frames, (long)in_stride, (long)out_stride, st);
    CUDA_CHECK(cudaEventRecord(m->ev1, st));
    m->timing_valid = true;
    return NAM_B200_OK;
  });
}

int nam_b200_process_f32(nam_b200_model* m, const float* in, float* out, int batch, int n_frames, int64_t in_stride,
                         int64_t out_stride)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    const int rc = check_process_args(m, in, out, batch, n_frames);
    if (rc != NAM_B200_OK)
      return rc;
    if (n_frames == 0)
      return NAM_B200_OK;
    const size_t ci = (size_t)m->spec.in_channels, co = (size_t)m->spec.out_channels;
    if ((size_t)in_stride < ci * n_frames || (size_t)out_stride < co * n_frames)
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, "stride smaller than channels x n_frames");
    const size_t row = (size_t)n_frames * sizeof(float);
    // Large WaveNet batches: pipeline the call in chunks of whole kernel waves so that the copies of chunk c+1 /
    // c-1 overlap the kernel of chunk c (the kernel is compute-bound; the copies would otherwise add ~18 %).
    const int chunk = wavenet_chunk_streams(m);
    if (chunk > 0 && batch >= 2 * chunk && (size_t)batch * row >= ((size_t)8 << 20))
    {
      const int n_chunks = (batch + chunk - 1) / chunk;
      if (!m->copy_in)
      {
        CUDA_CHECK(cudaStreamCreateWithFlags(&m->copy_in, cudaStreamNonBlocking));
        CUDA_CHECK(cudaStreamCreateWithFlags(&m->copy_out, cudaStreamNonBlocking));
      }
      while ((int)m->chunk_events.size() < 2 * n_chunks)
      {
        cudaEvent_t e;
        CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        m->chunk_events.push_back(e);
      }
      CUDA_CHECK(cudaEventRecord(m->ev0, m->stream));
      for (int c = 0; c < n_chunks; c++)
      {
        const int s0 = c * chunk, nb = std::min(chunk, batch - s0);
        float* din = m->d_in + (size_t)s0 * n_frames;
        float* dout = m->d_out + (size_t)s0 * n_frames;
        cudaEvent_t e_in = m->chunk_events[2 * c], e_k = m->chunk_events[2 * c + 1];
        CUDA_CHECK(cudaMemcpy2DAsync(din, row, in + (size_t)s0 * in_stride, (size_t)in_stride * sizeof(float), row,
                                     (size_t)nb, cudaMemcpyHostToDevice, m->copy_in));
        CUDA_CHECK(cudaEventRecord(e_in, m->copy_in));
        CUDA_CHECK(cudaStreamWaitEvent(m->stream, e_in, 0));
        launch_wavenet(m, din, dout, nb, n_frames, n_frames, n_frames, m->stream, s0);
        CUDA_CHECK(cudaEventRecord(e_k, m->stream));
        CUDA_CHECK(cudaStreamWaitEvent(m->copy_out, e_k, 0));
        CUDA_CHECK(cudaMemcpy2DAsync(out + (size_t)s0 * out_stride, (size_t)out_stride * sizeof(float), dout, row, row,
                                     (size_t)nb, cudaMemcpyDeviceToHost, m->copy_out));
      }
      m->t_base += (uint32_t)n_frames;
      m->streams_identical = false;
      CUDA_CHECK(cudaEventRecord(m->ev1, m->stream));
      CUDA_CHECK(cudaStreamSynchronize(m->copy_out));
      CUDA_CHECK(cudaStreamSynchronize(m->stream));
      m->timing_valid = true;
      return NAM_B200_OK;
    }
    // (multi-channel models: a stream's row is its channel planes back to back)
    CUDA_CHECK(cudaMemcpy2DAsync(m->d_in, ci * row, in, (size_t)in_stride * sizeof(float), ci * row, (size_t)batch,
                                 cudaMemcpyHostToDevice, m->stream));
    CUDA_CHECK(cudaEventRecord(m->ev0, m->stream));
    run_device(m, m->d_in, m->d_out, batch, n_frames, (long)(ci * n_frames), (long)(co * n_frames), m->stream);
    CUDA_CHECK(cudaEventRecord(m->ev1, m->stream));
    CUDA_CHECK(cudaMemcpy2DAsync(out, (size_t)out_stride * sizeof(float), m->d_out, co * row, co * row, (size_t)batch,
                                 cudaMemcpyDeviceToHost, m->stream));
    CUDA_CHECK(cudaStreamSynchronize(m->stream));
    m->timing_valid = true;
    return NAM_B200_OK;
  });
}

// ---- host-memory helpers ---------------------------------------------------------------------------------------------
// The host-buffer entries copy with cudaMemcpy2DAsync on side streams: with page-locked caller buffers the copies of
// chunk c+1 / c-1 run under the kernel of chunk c; with pageable buffers the driver stages every copy through its own
// bounce buffer and the overlap is lost (results are unaffected).  A host without the CUDA runtime pins through these.
int nam_b200_pin_host_buffer(void* ptr, int64_t bytes)
{
  if (!ptr || bytes <= 0)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null buffer or non-positive size");
  const cudaError_t e = cudaHostRegister(ptr, (size_t)bytes, cudaHostRegisterPortable);
  if (e != cudaSuccess && e != cudaErrorHostMemoryAlreadyRegistered)
  {
    cudaGetLastError();
    return fail(NAM_B200_ERR_CUDA, std::string("cudaHostRegister failed: ") + cudaGetErrorString(e));
  }
  cudaGetLastError();
  return NAM_B200_OK;
}
int nam_b200_unpin_host_buffer(void* ptr)
{
  if (!ptr)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null buffer");
  const cudaError_t e = cudaHostUnregister(ptr);
  if (e != cudaSuccess)
  {
    cudaGetLastError();
    return fail(NAM_B200_ERR_CUDA, std::string("cudaHostUnregister failed: ") + cudaGetErrorString(e));
  }
  return NAM_B200_OK;
}
/* 1 = page-locked (or device-accessible), 0 = pageable, < 0 = error */
int nam_b200_host_buffer_is_pinned(const void* ptr)
{
  cudaPointerAttributes a{};
  const cudaError_t e = cudaPointerGetAttributes(&a, ptr);
  if (e != cudaSuccess)
  {
    cudaGetLastError();
    return fail(NAM_B200_ERR_CUDA, std::string("cudaPointerGetAttributes failed: ") + cudaGetErrorString(e));
  }
  return a.type == cudaMemoryTypeUnregistered ? 0 : 1;
}

// ---- several GPUs behind one handle ------------------------------------------------------------------------------------
// The batch shards across devices (streams are independent: SURVEY.md 8e, no collective on the data path): one complete
// single-device handle per GPU, streams dealt out in contiguous blocks, one worker thread per GPU per call.
extern "C++" {
struct nam_b200_multi
{
  std::vector<std::unique_ptr<nam_b200_model>> parts;
  std::vector<int> first; // first stream of part i; first.back() = total streams
};

namespace
{
template <typename F>
int multi_for_each(nam_b200_multi* mm, F&& body) // body(part index) -> status; runs the parts concurrently
{
  const int n = (int)mm->parts.size();
  std::vector<int> rc(n, NAM_B200_OK);
  std::vector<std::string> msg(n);
  std::vector<std::thread> workers;
  for (int i = 0; i < n; i++)
    workers.emplace_back([&, i]() {
      rc[i] = body(i);
      if (rc[i] != NAM_B200_OK)
        msg[i] = g_last_error; // thread-local in the worker
    });
  for (auto& w : workers)
    w.join();
  for (int i = 0; i < n; i++)
    if (rc[i] != NAM_B200_OK)
      return fail(rc[i], "device " + std::to_string(mm->parts[i]->device) + ": " + msg[i]);
  return NAM_B200_OK;
}

int multi_create(const char* text_or_path, bool is_file, const nam_b200_options* opts, const int32_t* devices, int n_devices,
                 nam_b200_multi** out)
{
  if (!text_or_path || !out || n_devices < 1 || (n_devices > 0 && !devices))
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument or empty device list");
  nam_b200_options o;
  nam_b200_default_options(&o);
  if (opts)
    std::memcpy(&o, opts, std::min<size_t>(sizeof o, (size_t)std::max(opts->struct_size, 0)));
  o.struct_size = sizeof o;
  if (o.max_batch < n_devices)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "max_batch is smaller than the number of devices");
  std::unique_ptr<nam_b200_multi> mm(new nam_b200_multi());
  int s0 = 0;
  for (int i = 0; i < n_devices; i++)
  {
    const int s1 = (int)((int64_t)o.max_batch * (i + 1) / n_devices); // sharding.shard_bounds' rule
    nam_b200_options oi = o;
    oi.device = devices[i];
    oi.max_batch = s1 - s0;
    nam_b200_model* h = nullptr;
    const int rc = is_file ? nam_b200_create_from_file(text_or_path, &oi, &h) : nam_b200_create_from_json(text_or_path, &oi, &h);
    if (rc != NAM_B200_OK)
      return rc;
    mm->parts.emplace_back(h);
    mm->first.push_back(s0);
    s0 = s1;
  }
  mm->first.push_back(s0);
  *out = mm.release();
  return NAM_B200_OK;
}
} // namespace
} // extern "C++"

int nam_b200_multi_create_from_file(const char* nam_path, const nam_b200_options* opts, const int32_t* devices, int n_devices,
                                    nam_b200_multi** out)
{
  return multi_create(nam_path, true, opts, devices, n_devices, out);
}
int nam_b200_multi_create_from_json(const char* nam_json_text, const nam_b200_options* opts, const int32_t* devices,
                                    int n_devices, nam_b200_multi** out)
{
  return multi_create(nam_json_text, false, opts, devices, n_devices, out);
}
void nam_b200_multi_destroy(nam_b200_multi* mm)
{
  delete mm;
}
int nam_b200_multi_device_count(const nam_b200_multi* mm)
{
  return mm ? (int)mm->parts.size() : 0;
}
int nam_b200_multi_shard(const nam_b200_multi* mm, int part, int32_t* device, int32_t* first_stream, int32_t* n_streams)
{
  if (!mm || part < 0 || part >= (int)mm->parts.size())
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "no such part");
  if (device)
    *device = mm->parts[part]->device;
  if (first_stream)
    *first_stream = mm->first[part];
  if (n_streams)
    *n_streams = mm->first[part + 1] - mm->first[part];
  return NAM_B200_OK;
}
int nam_b200_multi_reset(nam_b200_multi* mm, double sample_rate, int max_frames)
{
  if (!mm)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null handle");
  return multi_for_each(mm, [&](int i) { return nam_b200_reset(mm->parts[i].get(), sample_rate, max_frames); });
}
int nam_b200_multi_process_f32(nam_b200_multi* mm, const float* in, float* out, int batch, int n_frames, int64_t in_stride,
                               int64_t out_stride)
{
  if (!mm || !in || !out)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument");
  if (batch < 1 || batch > mm->first.back())
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "batch outside [1, max_batch]");
  return multi_for_each(mm, [&](int i) {
    const int s0 = mm->first[i], nb = std::min(mm->first[i + 1], batch) - s0;
    if (nb <= 0)
      return (int)NAM_B200_OK;
    return nam_b200_process_f32(mm->parts[i].get(), in + (size_t)s0 * in_stride, out + (size_t)s0 * out_stride, nb, n_frames,
                                in_stride, out_stride);
  });
}

int nam_b200_process_f32_planar(nam_b200_model* m, const float* const* input, float* const* output, int n_frames)
{
  return process_planar<float>(m, input, output, n_frames);
}

int nam_b200_process_f64_planar(nam_b200_model* m, const double* const* input, double* const* output, int n_frames)
{
  return process_planar<double>(m, input, output, n_frames);
}

int nam_b200_has_tensor_core_kernel(void)
{
  return 0; // no tensor-core WaveNet kernel on sm_90a
}

int nam_b200_set_reserved_sms(nam_b200_model* m, int n_sms)
{
  if (!m || n_sms < 0)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null model handle or negative count");
  m->reserved_sms = n_sms;
  for (auto& sub : m->subs)
    sub->reserved_sms = n_sms;
  return NAM_B200_OK;
}

int nam_b200_set_fast_tanh(nam_b200_model* m, int enabled)
{
  if (!m)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null model handle");
  m->fast_tanh_runtime = enabled ? 1 : 0; // only the LSTM kernel reads it (lstm.cpp:48)
  for (auto& sub : m->subs)
    sub->fast_tanh_runtime = m->fast_tanh_runtime;
  return NAM_B200_OK;
}

int nam_b200_set_slimmable_size(nam_b200_model* m, double value)
{
  if (!m)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null model handle");
  if (m->active_sub < 0)
    return fail(NAM_B200_ERR_UNSUPPORTED, "model is not slimmable (not a SlimmableContainer)");
  // ContainerModel::_get_index_for_slimmable_size / SetSlimmableSize (container.cpp:88-122)
  int idx = (int)m->subs.size() - 1;
  for (size_t i = 0; i < m->subs.size(); i++)
    if (value < m->spec.submodels[i].max_value)
    {
      idx = (int)i;
      break;
    }
  if (idx == m->active_sub)
    return NAM_B200_OK;
  if (m->is_reset)
  {
    // the newly selected sub-model is reset (and prewarmed) before it becomes the active one
    const double sr = m->ext_sample_rate;
    const int rc = nam_b200_reset(m->subs[(size_t)idx].get(), sr, m->max_frames);
    if (rc != NAM_B200_OK)
      return rc;
  }
  m->active_sub = idx;
  return 1; // switched
}

int nam_b200_slimmable_breakpoints(const nam_b200_model* m, double* out, int capacity)
{
  if (!m)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null model handle");
  if (m->active_sub < 0)
    return 0;
  const int n = (int)m->subs.size() - 1; // container.cpp:124-133
  for (int i = 0; i < n && i < capacity && out; i++)
    out[i] = m->spec.submodels[(size_t)i].max_value;
  return n;
}

int nam_b200_synchronize(nam_b200_model* m)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    CUDA_CHECK(cudaStreamSynchronize(m->stream));
    return NAM_B200_OK;
  });
}

int64_t nam_b200_launch_count(const nam_b200_model* m)
{
  if (!m)
    return -1;
  int64_t n = m->launches;
  for (const auto& sub : m->subs)
    n += sub->launches;
  return n;
}

double nam_b200_last_kernel_ms(nam_b200_model* m)
{
  m = active_model(m);
  if (!m || !m->timing_valid)
    return -1.0;
  cudaSetDevice(m->device);
  if (cudaEventSynchronize(m->ev1) != cudaSuccess)
    return -1.0;
  float ms = 0.0f;
  if (cudaEventElapsedTime(&ms, m->ev0, m->ev1) != cudaSuccess)
    return -1.0;
  return (double)ms;
}

double nam_b200_measure_fp32_tflops(int device, int /*use_ffma2: no packed FP32 FMA on sm_90*/)
{
  try
  {
    if (device >= 0)
      CUDA_CHECK(cudaSetDevice(device));
    cudaDeviceProp prop{};
    int dev = 0;
    CUDA_CHECK(cudaGetDevice(&dev));
    CUDA_CHECK(cudaGetDeviceProperties(&prop, dev));
    float* d = nullptr;
    CUDA_CHECK(cudaMalloc(&d, 4));
    cudaEvent_t e0, e1;
    CUDA_CHECK(cudaEventCreate(&e0));
    CUDA_CHECK(cudaEventCreate(&e1));
    const int iters = 4096, blocks = prop.multiProcessorCount * 8, threads = 256;
    double best = 0.0;
    for (int rep = 0; rep < 5; rep++)
    {
      CUDA_CHECK(cudaEventRecord(e0));
      fma_peak_kernel<<<blocks, threads>>>(d, iters, 1.0f);
      CUDA_CHECK(cudaEventRecord(e1));
      CUDA_CHECK(cudaEventSynchronize(e1));
      float ms = 0.0f;
      CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
      const double flops = 2.0 * 16.0 * (double)iters * blocks * threads;
      best = std::max(best, flops / (ms * 1e-3) / 1e12);
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaFree(d);
    return best;
  }
  catch (const std::exception& ex)
  {
    fail(NAM_B200_ERR_CUDA, ex.what());
    return -1.0;
  }
}

} // extern "C"
