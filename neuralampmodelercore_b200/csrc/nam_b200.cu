// nam_b200.cu -- C ABI of libnam_b200.so (include/nam_b200.h): model handles, device state,
// kernel launches.  Host code is C++; every hot-path operation is a hand-written sm_90a kernel
// (wavenet_fused.cuh, and the LSTM / Linear kernels below).  There is deliberately no CPU
// fallback anywhere in this file.
#include "../../include/nam_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstddef>
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
#include "stream_state.cuh"
#include "resample.h"
#include "resample.cuh"

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
  // slot table (nullptr: position b is state row b): position b uses state row slots[b].stream; in / out stay by position
  const StreamRef* slots;
  // model bank (the BANK instantiations; they always get a table): position b runs model slots[b].model, whose blob starts
  // at weights + model * weight_stride.  bank_copies: the model copies lstm_group_kernel's shared memory holds.
  long weight_stride;
  int bank_copies;
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

// BANK (model banks): the weights of one model fill shared memory, so the CTA runs one pass of the chunk loop per distinct
// model among its positions, that model's blob staged for the pass; a position outside the pass runs 0 frames in it (its
// state stays as it is, it writes no output).  Positions of one model in adjacent slots keep a CTA at one pass; round-robin
// binding of 64 or more models costs up to 64.  Each stream's arithmetic is the ordinary instantiation's.
template <bool BANK = false>
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

  if constexpr (!BANK)
    for (int i = tid; i < p.n_weight_floats; i += kLstmThreads)
      sw[i] = __ldg(p.weights + i);
  const int stream = blockIdx.x * kLstmThreads + tid;
  const bool active = stream < p.batch;
  const size_t row = p.slots ? (size_t)p.slots[active ? stream : 0].stream : (size_t)stream;
  const int n_state = p.num_layers * 2 * H;
  if (active)
    for (int i = 0; i < n_state; i++)
      sstate[i * kLstmThreads + tid] = p.state[row * p.state_stride + i];
  const int stream0 = blockIdx.x * kLstmThreads;
  // BANK: s_model[s] = the model of position s (-1 beyond the batch), s_first[s] = the first position of that model
  __shared__ int s_model[BANK ? kLstmThreads : 1], s_first[BANK ? kLstmThreads : 1];
  if constexpr (BANK)
  {
    s_model[tid] = active ? p.slots[stream].model : -1;
    __syncthreads();
    int first = tid;
    for (int s = tid - 1; s >= 0; s--)
      first = s_model[s] == s_model[tid] ? s : first;
    s_first[tid] = s_model[tid] < 0 ? -1 : first;
  }
  __syncthreads();

  // one pass per distinct model, led by its first position (an ordinary CTA: one pass over every position)
  for (int lead = 0; lead < (BANK ? kLstmThreads : 1); lead++)
  {
    if constexpr (BANK)
    {
      if (s_first[lead] != lead) // (uniform: shared)
        continue;
      const float* src = p.weights + (size_t)s_model[lead] * p.weight_stride;
      for (int i = tid; i < p.n_weight_floats; i += kLstmThreads)
        sw[i] = __ldg(src + i); // (the previous pass's last barrier ordered its reads before these writes)
    }
    // frames of the CTA's position s in this pass (slot table: the stream's own count; 0 beyond the batch and, in a bank, for
    // another model's position); the chunk loop holds barriers, so it runs to the pass's longest stream
    auto frames_of = [&](int s) -> int {
      const int b = stream0 + s;
      if (BANK && s_model[s] != s_model[lead])
        return 0;
      return b >= p.batch ? 0 : p.slots ? p.slots[b].frames : p.n_frames;
    };
    int n_cta = 0;
    for (int s = 0; s < kLstmThreads; s++)
      n_cta = max(n_cta, frames_of(s));
    const int n_me = frames_of(tid);
    for (int t0 = 0; t0 < n_cta; t0 += kLstmChunk)
    {
      // coalesced load of the [streams x chunk] input tile
      for (int idx = tid; idx < kLstmThreads * kLstmChunk; idx += kLstmThreads)
      {
        const int s = idx / kLstmChunk, f = idx - s * kLstmChunk;
        float v = 0.0f;
        if (t0 + f < frames_of(s))
          v = __ldg(p.in + (size_t)(stream0 + s) * p.in_stride + t0 + f);
        sio[s * (kLstmChunk + 1) + f] = v;
      }
      __syncthreads();
      const int tc = min(kLstmChunk, n_me - t0); // this thread's frames in the chunk (<= 0: its stream has ended)
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
        if (t0 + f < frames_of(s) && p.out_ch == 1 && p.in_ch == 1)
          p.out[(size_t)(stream0 + s) * p.out_stride + t0 + f] = sout[s * (kLstmChunk + 1) + f];
      }
      __syncthreads();
    }
  }
  if (active)
    for (int i = 0; i < n_state; i++)
      p.state[row * p.state_stride + i] = sstate[i * kLstmThreads + tid];
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
  // slot table (nullptr: position b is row b of `state`): position b uses row slots[b].stream of `state`, or of `state_alt`
  // when slots[b].alt -- each stream reads the buffer it was last written to and the update writes the other one
  const StreamRef* slots;
  float* __restrict__ state_alt;
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
  const float* st = p.slots ? (p.slots[stream].alt ? p.state_alt : p.state) + (size_t)p.slots[stream].stream * p.state_stride
                            : p.state + (size_t)stream * p.state_stride;
  const int n = p.slots ? p.slots[stream].frames : p.n_frames; // this stream's frames
  for (int i = tid; i < hist + kLinThreads; i += kLinThreads)
  {
    const int t = t0 - hist + i; // frame index relative to this call
    float v = 0.0f;
    if (t >= 0)
      v = (t < n) ? __ldg(xin + t) : 0.0f;
    else
      v = st[hist + t]; // t in [-hist, 0): state holds frames -hist..-1
    sx[i] = v;
  }
  __syncthreads();
  const int t = t0 + tid;
  if (t < n)
  {
    // oldest tap first, like the reference's dot over the reversed impulse (linear.cpp:71-74,184-186)
    float acc = 0.0f;
    for (int j = hist; j >= 0; j--)
      acc = fmaf(sw[j], sx[hist + tid - j], acc);
    p.out[(size_t)stream * p.out_stride + t] = p.bias + acc;
  }
}

// new_state = last (rf-1) samples of [old_state | in[0:n)] (slot table: into the other buffer of each stream's pair, n the
// stream's own count; a stream with n == 0 keeps its history where it is, and the host counts no flip for it)
__global__ void linear_update_state_kernel(const LinearKernelParams p, float* __restrict__ new_state)
{
  const int hist = p.rf - 1;
  const int stream = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= hist)
    return;
  int n = p.n_frames;
  const float* old_st = p.state + (size_t)stream * p.state_stride;
  float* new_st = new_state + (size_t)stream * p.state_stride;
  if (p.slots)
  {
    const StreamRef r = p.slots[stream];
    if (r.frames == 0)
      return;
    n = r.frames;
    old_st = (r.alt ? p.state_alt : p.state) + (size_t)r.stream * p.state_stride;
    new_st = (r.alt ? p.state : p.state_alt) + (size_t)r.stream * p.state_stride;
  }
  const int t = n - hist + i; // relative frame index of new history slot i
  float v;
  if (t >= 0)
    v = p.in[(size_t)stream * p.in_stride + t];
  else
    v = old_st[hist + t];
  new_st[i] = v;
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

// A module the handle compiled at run time (jit_spec.cpp), loaded from its cubin: unloaded when its owner goes away or
// loads another one.
class JitModule
{
public:
  JitModule() = default;
  JitModule(const JitModule&) = delete;
  JitModule& operator=(const JitModule&) = delete;
  ~JitModule() { unload(); }
  explicit operator bool() const { return lib_ != nullptr; }
  void unload()
  {
    if (lib_)
      cudaLibraryUnload(lib_);
    lib_ = nullptr;
  }
  // Loads `cubin` in place of the module held.  Returns "" or what failed.
  std::string load(const std::vector<char>& cubin)
  {
    unload();
    const cudaError_t e = cudaLibraryLoadData(&lib_, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
    if (e != cudaSuccess)
      lib_ = nullptr;
    return failed(e, "cudaLibraryLoadData");
  }
  // Entry point `name` -> *k, allowed `smem` bytes of dynamic shared memory (0: none); with `ctas_per_sm`, also its
  // resident CTAs of `threads` threads per SM.  Returns "" or what failed (*k = nullptr).
  std::string kernel(cudaKernel_t* k, const char* name, size_t smem = 0, int threads = 0, int* ctas_per_sm = nullptr) const
  {
    std::string why = failed(cudaLibraryGetKernel(k, lib_, name), "cudaLibraryGetKernel");
    if (why.empty() && smem > 0)
      why = failed(cudaFuncSetAttribute((const void*)*k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                   "cudaFuncSetAttribute");
    if (why.empty() && ctas_per_sm)
      why = failed(cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas_per_sm, (const void*)*k, threads, smem),
                   "cudaOccupancyMaxActiveBlocksPerMultiprocessor");
    if (!why.empty())
      *k = nullptr;
    return why;
  }

private:
  // "" or "<call> failed: <error>".  The error is cleared, so that a later launch check does not report it.
  static std::string failed(cudaError_t e, const char* call)
  {
    if (e == cudaSuccess)
      return "";
    cudaGetLastError();
    return std::string(call) + " failed: " + cudaGetErrorString(e);
  }
  cudaLibrary_t lib_ = nullptr;
};

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
  JitModule spec_lib; // (or the LSTM's, or the general kernel's)
  JitModule spec_lib_extra; // second program of the model: the 128- / 256-frame short-call entry points
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
  JitModule lat_lib;
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
  // per-stream state control (stream_state.cuh)
  std::vector<uint32_t> stream_clock; // t_base at which each stream's history ends (streams left out of calls fall behind)
  std::vector<uint32_t> stream_flips; // Linear: lin_flips when the stream's history was written (parity picks the buffer)
  uint32_t lin_flips = 0; // Linear: d_state / d_state_tmp swaps so far
  std::vector<StateSegDesc> state_descs; // record segments -> device layout, built at creation
  std::vector<StateChunk> state_chunks;
  StateSegDesc* d_state_descs = nullptr;
  StateChunk* d_state_chunks = nullptr;
  long record_floats = 0; // payload floats of one record
  StateRecordHeader record_header{};
  std::string state_error; // non-empty: the stream-state calls are refused with this reason
  unsigned char* d_fresh = nullptr; // WaveNet / ConvNet / Linear: the record of a stream straight after nam_b200_reset
  StreamRef* d_refs = nullptr; // stream lists of pack / unpack / row-copy launches
  // slot tables of process calls (nam_b200_process_streams_f32, and contiguous calls over a stream that sat out calls):
  // position i of the call -> state row, clock and Linear buffer.  The host copy is rebuilt per call; the device copy
  // (max_batch entries) is rewritten only once the previous table call's kernels, on whichever CUDA stream, are done with it
  std::vector<StreamRef> h_slots;
  StreamRef* d_slots = nullptr;
  cudaEvent_t slots_free = nullptr; // recorded after the last launch that reads d_slots
  bool slots_used = false;
  int n_out_of_phase = 0; // streams whose history does not end at t_base (Linear: or sits in the other buffer)
  size_t refs_capacity = 0;
  // model bank (nam_b200_create_bank_*): bank_size WaveNets of one WaveNetPlan, or LSTMs of one shape, each stream
  // bound to one of them.  d_weights holds their blobs weight_stride floats apart, d_head_scales the WaveNets' output
  // scales, d_bank_headers their record headers.  State rows max_batch + k (k < bank_size) are the models' fresh
  // rows: reset prewarms them together (a WaveNet bank then copies them out; an LSTM's streams keep their running state);
  // reset_streams / assign_streams copy them.  Their histories end at fresh_clock.  An LSTM bank's rows were prewarmed in
  // the fast-tanh regime rows_fast_tanh; a switch rebuilds them before the next copy.
  // is_bank is set by create_bank alone (a bank of bank_capacity > 1 is one even while bank_size == 1).  Everything above
  // is sized for bank_capacity models at creation, so nam_b200_bank_add_models never moves what live streams use.
  // Ordinary handles: is_bank false, bank_size and bank_capacity 1, stream_model all 0, no extra rows.
  bool is_bank = false;
  int bank_size = 1;
  int bank_capacity = 1;
  std::vector<ModelSpec> bank_specs; // model k's document (bank_size entries; bank_specs[0] is `spec`'s twin)
  std::vector<StateRecordHeader> bank_headers;
  std::vector<int32_t> stream_model;
  long weight_stride = 0;
  float* d_head_scales = nullptr;
  uint32_t* d_bank_headers = nullptr;
  uint32_t fresh_clock = 0;
  int rows_fast_tanh = -1;
  unsigned char* d_xfer = nullptr; // staging of host records, scratch rows of copies and LSTM prewarms
  size_t xfer_bytes = 0;
  // staging
  float* d_in = nullptr;
  float* d_out = nullptr;
  size_t staging_floats = 0;
  float* h_pin = nullptr; // pinned, device-mapped scratch for the planar (single stream) entry points
  float* h_pin_dev = nullptr; // its device-side address
  size_t h_pin_floats = 0;
  double flops_per_frame = 0.0;

  // sample-rate conversion (options.resample, resample.cuh), set up by reset when the host rate differs from the model's.
  // Per stream, one row of rs_stride floats: in_channels x H_up host inputs, then out_channels x H_dn model outputs; row
  // max_batch stays zero (reset_streams copies it).  phase[s] = h mod M of stream s.  max_frames is then the model's
  // (ceil(host_max_frames L / M)); the process entries check host frames against host_max_frames.
  struct Resampler
  {
    bool active = false;
    ResamplerDesign design;
    int H_up = 0, H_dn = 0, rs_stride = 0;
    int host_max_frames = 0;
    std::vector<uint32_t> phase;
    std::vector<RsPos> h_pos;
    float* d_taps = nullptr; // phase tables: host -> model ([T_up][L]), then model -> host ([T_dn][M])
    float* d_hist = nullptr; // (max_batch + 1) rows
    float* d_x = nullptr; // model-rate input of a call, [position][in_channels][n_max]
    float* d_z = nullptr; // model-rate output, [position][out_channels][n_max]
    RsPos* d_pos = nullptr;
    cudaEvent_t pos_free = nullptr; // recorded after the last launch that reads d_pos
    bool pos_used = false;
  } rs;

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
    if (d_tile_flags)
      cudaFree(d_tile_flags);
    if (d_hist)
      cudaFree(d_hist);
    if (d_state)
      cudaFree(d_state);
    if (d_state_tmp)
      cudaFree(d_state_tmp);
    if (d_state_descs)
      cudaFree(d_state_descs);
    if (d_state_chunks)
      cudaFree(d_state_chunks);
    if (d_fresh)
      cudaFree(d_fresh);
    if (d_refs)
      cudaFree(d_refs);
    if (d_slots)
      cudaFree(d_slots);
    if (slots_free)
      cudaEventDestroy(slots_free);
    if (d_xfer)
      cudaFree(d_xfer);
    if (d_head_scales)
      cudaFree(d_head_scales);
    if (d_bank_headers)
      cudaFree(d_bank_headers);
    if (d_in)
      cudaFree(d_in);
    if (d_out)
      cudaFree(d_out);
    for (void* p : {(void*)rs.d_taps, (void*)rs.d_hist, (void*)rs.d_x, (void*)rs.d_z, (void*)rs.d_pos})
      if (p)
        cudaFree(p);
    if (rs.pos_free)
      cudaEventDestroy(rs.pos_free);
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

// The channel pairs the fused kernels are compiled for: (C0, C1) = the padded channels of array 0 and array 1 (0: one array)
constexpr int kChannelPairs[][2] = {{4, 0}, {8, 0}, {16, 0}, {4, 4}, {4, 8}, {4, 16}, {8, 4}, {8, 8}, {8, 16}, {16, 4}, {16, 8}, {16, 16}};
constexpr int kNumChannelPairs = (int)(sizeof(kChannelPairs) / sizeof(kChannelPairs[0]));
template <int V>
using IntC = std::integral_constant<int, V>;

// f(IntC<C0>, IntC<C1>) for the listed pair (c0, c1); `kind` names the kernel in the error for a pair outside the list
template <int P = 0, typename F>
auto with_channel_pair(int c0, int c1, const char* kind, const F& f) -> decltype(f(IntC<4>{}, IntC<0>{}))
{
  if constexpr (P == kNumChannelPairs)
    throw std::runtime_error(std::string("no ") + kind + " WaveNet kernel for channel pair " + std::to_string(c0) + "/"
                             + std::to_string(c1));
  else
  {
    if (c0 == kChannelPairs[P][0] && c1 == kChannelPairs[P][1])
      return f(IntC<kChannelPairs[P][0]>{}, IntC<kChannelPairs[P][1]>{});
    return with_channel_pair<P + 1>(c0, c1, kind, f);
  }
}
// f(IntC<g>) for g in [0, N), the last one for any g outside
template <int N, int G = 0, typename F>
auto with_index(int g, const F& f) -> decltype(f(IntC<0>{}))
{
  if constexpr (G + 1 < N)
    if (g != G)
      return with_index<N, G + 1>(g, f);
  return f(IntC<G>{});
}

// One launch of the fused kernel; calls with a slot table run its TBL instantiation
template <int C0, int C1, int S, int NT, int MINB, int LQ, bool LS>
void launch_fused(nam_b200_model* m, const WaveNetKernelParams& kp, int grid, size_t smem, cudaStream_t st)
{
  auto kern = kp.slots ? wavenet_fused_kernel<C0, C1, S, NT, MINB, LQ, LS, true> : wavenet_fused_kernel<C0, C1, S, NT, MINB, LQ, LS>;
  ensure_max_dynamic_smem(reinterpret_cast<const void*>(kern), m->device, 227 * 1024);
  if constexpr (LS)
  {
    // The tiles spin on each other's flags, so they must all be resident at once: a cooperative launch is
    // gang-scheduled (it starts only when the whole grid fits), which keeps two such launches from different handles
    // from starving each other.
    void* args[] = {const_cast<void*>(static_cast<const void*>(&kp))};
    CUDA_CHECK(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(kern), dim3((unsigned)grid), dim3(NT), args, smem, st));
  }
  else
  {
    kern<<<grid, NT, smem, st>>>(kp);
    CUDA_CHECK(cudaGetLastError());
  }
}

// CTAs per SM of the fused kernel: the lower of its two instantiations, so that the co-residency the tile-parallel modes
// rely on holds for both
template <int C0, int C1, int S, int NT, int MINB, int LQ, bool LS>
int occupancy_fused(size_t smem)
{
  int best = 1 << 30;
  for (auto kern : {wavenet_fused_kernel<C0, C1, S, NT, MINB, LQ, LS>, wavenet_fused_kernel<C0, C1, S, NT, MINB, LQ, LS, true>})
  {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, NT, smem) != cudaSuccess)
      return 1;
    best = std::min(best, n);
  }
  return best > 0 ? best : 1;
}

void launch_wavenet_dispatch(int c0, int c1, int geom, nam_b200_model* m, const WaveNetKernelParams& kp, int grid,
                             size_t smem, cudaStream_t st)
{
  with_channel_pair(c0, c1, "fused", [&](auto C0, auto C1) {
    with_index<4>(geom, [&](auto g) {
      constexpr WnGeometry G = kWnGeom[decltype(g)::value];
      launch_fused<decltype(C0)::value, decltype(C1)::value, kWnS, G.nt, G.min_ctas, G.lq, false>(m, kp, grid, smem, st);
    });
  });
}
int occupancy_wavenet_dispatch(int c0, int c1, int geom, size_t smem)
{
  return with_channel_pair(c0, c1, "fused", [&](auto C0, auto C1) {
    return with_index<4>(geom, [&](auto g) {
      constexpr WnGeometry G = kWnGeom[decltype(g)::value];
      return occupancy_fused<decltype(C0)::value, decltype(C1)::value, kWnS, G.nt, G.min_ctas, G.lq, false>(smem);
    });
  });
}

void launch_wavenet_ls_dispatch(int c0, int c1, int geom, nam_b200_model* m, const WaveNetKernelParams& kp, int grid,
                                size_t smem, cudaStream_t st)
{
  with_channel_pair(c0, c1, "fused", [&](auto C0, auto C1) {
    with_index<kLsGeoms>(geom, [&](auto g) {
      constexpr LsGeometry G = kLsGeom[decltype(g)::value];
      launch_fused<decltype(C0)::value, decltype(C1)::value, G.s, G.nt, G.min_ctas, G.lq, true>(m, kp, grid, smem, st);
    });
  });
}
int occupancy_wavenet_ls_dispatch(int c0, int c1, int geom, size_t smem)
{
  return with_channel_pair(c0, c1, "fused", [&](auto C0, auto C1) {
    return with_index<kLsGeoms>(geom, [&](auto g) {
      constexpr LsGeometry G = kLsGeom[decltype(g)::value];
      return occupancy_fused<decltype(C0)::value, decltype(C1)::value, G.s, G.nt, G.min_ctas, G.lq, true>(smem);
    });
  });
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
    auto kern = kp.slots ? wavenet_lat2_kernel<C0, C1, 2, true> : wavenet_lat2_kernel<C0, C1, 2>;
    ensure_max_dynamic_smem(reinterpret_cast<const void*>(kern), m->device, 200 * 1024); // (+ 520 B of static mbarriers)
    kern<<<kp.batch, 256, smem, st>>>(kp);
  }
  else
  {
    auto kern = kp.slots ? wavenet_lat2_kernel<C0, C1, 4, true> : wavenet_lat2_kernel<C0, C1, 4>;
    ensure_max_dynamic_smem(reinterpret_cast<const void*>(kern), m->device, 200 * 1024);
    kern<<<kp.batch, 512, smem, st>>>(kp);
  }
  CUDA_CHECK(cudaGetLastError());
}
void launch_wavenet_lat2_dispatch(int c0, int c1, nam_b200_model* m, const WaveNetKernelParams& kp, int fw, size_t smem,
                                  cudaStream_t st)
{
  with_channel_pair(c0, c1, "low-latency", [&](auto C0, auto C1) {
    launch_wavenet_lat2_variant<decltype(C0)::value, decltype(C1)::value>(m, kp, fw, smem, st);
  });
}

constexpr int kSmallNt = 128, kSmallLq = 7;
void launch_wavenet_small_dispatch(int c0, int c1, nam_b200_model* m, const WaveNetKernelParams& kp, int grid, size_t smem,
                                   cudaStream_t st)
{
  with_channel_pair(c0, c1, "fused", [&](auto C0, auto C1) {
    launch_fused<decltype(C0)::value, decltype(C1)::value, 1, kSmallNt, 3, kSmallLq, false>(m, kp, grid, smem, st);
  });
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
// Geometry of the specialised kernel for a handle of `max_batch` streams (its tile is the model's: spec_tile_geometry).
// Streams per CTA of the short-call entry point: the count that fills whole waves of 2 CTAs per SM best (4096 streams on
// 132 SMs: 8 per CTA = 512 CTAs = 1.94 waves, 7 per CTA = 586 = 2.22 waves).
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

// Does this handle want a model-specialised throughput kernel?  Required (jit = 1), or automatic / preferred on a throughput
// handle (max_batch >= 256), where one compilation pays for itself within the first calls.  $NAM_B200_JIT=0/1 overrides
// "automatic".
bool jit_wanted(const nam_b200_model* m)
{
  const int mode = jit_mode(m);
  return mode == 1 || ((mode == 0 || mode == 3) && m->opts.max_batch >= 256);
}

// The wanted model-specialised kernel cannot be had (`why`): the handle runs the precompiled kernels and its note says why.
// jit = 1 fails creation instead: NAM_B200_ERR_MODEL when the kernel did not compile, NAM_B200_ERR_CUDA when it did not load.
void jit_unavailable(nam_b200_model* m, const std::string& why, bool compiled)
{
  m->spec_lib.unload();
  m->spec_lib_extra.unload();
  m->spec_kernel = m->gen_spec_kernel = nullptr;
  for (auto& sv : m->spec_short)
    sv = nam_b200_model::SpecShort{};
  m->spec_state = -1;
  m->spec_note = why;
  if (jit_mode(m) == 1)
  {
    if (!compiled)
      throw std::runtime_error("model-specialised kernel unavailable: " + why);
    throw CudaError(why);
  }
}

std::string jit_loaded_note(const SpecBuild& b)
{
  return b.from_cache ? "cubin from cache" : "compiled in " + std::to_string(b.compile_seconds) + " s";
}

// The fused WaveNet family's specialised kernel (wavenet_spec.cuh), for handles with the default kernel geometry.  Its
// short-call entry points are optional: one that does not load only leaves its calls to the other kernels.
void setup_spec_kernel(nam_b200_model* m)
{
  if (!jit_wanted(m) || m->opts.kernel_geometry != 0)
    return;
  const SpecBuild b = build_spec_kernel(m->plan, spec_geometry_for(m->opts.max_batch, m->sm_count));
  m->spec_geom = b.geom;
  m->spec_smem = b.smem_bytes();
  std::string why = b.ok ? m->spec_lib.load(b.cubin) : b.why_not;
  if (why.empty())
    why = m->spec_lib.kernel(&m->spec_kernel, spec_kernel_name(), m->spec_smem, b.geom.nt, &m->spec_ctas_per_sm);
  if (why.empty() && m->spec_ctas_per_sm < 1)
    why = "the specialised kernel does not fit on an SM";
  if (!why.empty())
    return jit_unavailable(m, why, b.ok);
  if (b.has_short)
  {
    const char* const names[3] = {"wavenet_spec_short_kernel", "wavenet_spec_short128_kernel", "wavenet_spec_short256_kernel"};
    const int fqs[3] = {64, 128, 256}, qs[3] = {b.geom.short_streams, b.geom.short128_streams, b.geom.short256_streams};
    if (!b.cubin_extra.empty())
      m->spec_lib_extra.load(b.cubin_extra);
    for (int v = 0; v < 3; v++)
    {
      nam_b200_model::SpecShort& sv = m->spec_short[v];
      sv = nam_b200_model::SpecShort{};
      const JitModule& lib = (v == 0) ? m->spec_lib : m->spec_lib_extra;
      if (!lib)
        continue;
      sv.fq = fqs[v];
      sv.q = qs[v];
      sv.smem = (size_t)b.max_planes * sv.fq * sv.q * 16;
      if (!lib.kernel(&sv.kernel, names[v], sv.smem, sv.fq * sv.q, &sv.ctas_per_sm).empty() || sv.ctas_per_sm < 1)
        sv.kernel = nullptr;
    }
  }
  m->spec_state = 1;
  m->spec_note = jit_loaded_note(b);
}

// reset(): plugin-style handles (few streams, maxBufferSize <= 128) get the low-latency kernel for calls of up to
// 64 / 128 frames.  Wanted when jit is "required" or "preferred" (the C++ shim's default), never by the automatic policy.
// It never fails creation: without it the precompiled short-call geometries serve the handle.
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
  const SpecBuild b = build_lat_kernel(m->plan, fw);
  m->lat_smem = lat_smem_bytes(m->plan, 32 * fw);
  std::string why = b.why_not;
  if (b.ok)
  {
    std::string err = m->lat_lib.load(b.cubin);
    if (err.empty())
      err = m->lat_lib.kernel(&m->lat_kernel, "wavenet_lat_kernel", m->lat_smem);
    if (!err.empty())
      why = "loading the low-latency kernel failed: " + err;
  }
  if (!why.empty())
  {
    m->lat_lib.unload();
    m->lat_kernel = nullptr;
    m->lat_state = -1;
    m->lat_note = why;
    return;
  }
  m->lat_frames = 32 * fw;
  m->lat_threads = b.geom.nt;
  m->lat_state = 1;
  m->lat_note = jit_loaded_note(b);
}

// The parameter of the model-specialised kernels for one call: rows from `state` (the table's rows when `slots`), the call's
// buffers, strides, batch and frames, at the handle's clock
JitParams jit_params(const nam_b200_model* m, float* state, const float* d_in, float* d_out, long in_stride, long out_stride,
                     int batch, int n_frames, const StreamRef* slots)
{
  return JitParams{state,      m->state_stride, d_in, d_out, in_stride, out_stride, batch, n_frames, m->t_base, slots,
                   m->d_weights, m->weight_stride};
}

void launch_wavenet_lat(nam_b200_model* m, const JitParams& jp, cudaStream_t st)
{
  // single-stream calls ring the doorbell in mapped host memory (process_planar spins on it instead of synchronising)
  unsigned* flag = (jp.batch == 1 && m->h_flag_dev != nullptr) ? m->h_flag_dev : nullptr;
  if (flag)
    m->flag_seq++;
  LatParams lp{jp, flag, m->flag_seq};
  m->flag_pending = flag != nullptr;
  void* args[] = {&lp};
  CUDA_CHECK(cudaLaunchKernel((const void*)m->lat_kernel, dim3(jp.batch), dim3(m->lat_threads), args, m->lat_smem, st));
}

void launch_wavenet_spec(nam_b200_model* m, JitParams jp, cudaStream_t st)
{
  void* args[] = {&jp};
  int grid = std::min(jp.batch, m->spec_ctas_per_sm * std::max(1, m->sm_count - m->reserved_sms));
  if (grid < 1)
    grid = 1;
  CUDA_CHECK(cudaLaunchKernel((const void*)m->spec_kernel, dim3(grid), dim3(m->spec_geom.nt), args, m->spec_smem, st));
}

void launch_wavenet(nam_b200_model* m, const JitParams& call, cudaStream_t st)
{
  JitParams jp = call;
  const int batch = call.batch, n_frames = call.n_frames;
  if (m->use_generic && m->gen_spec_kernel != nullptr && m->opts.kernel_geometry == 0)
  {
    void* args[] = {&jp};
    // (a bank's shape-compiled kernel stages each stream's blob in dynamic shared memory)
    const size_t smem = m->is_bank ? (size_t)m->weight_stride * sizeof(float) : 0;
    CUDA_CHECK(cudaLaunchKernel((const void*)m->gen_spec_kernel, dim3(std::max(1, std::min(batch, 16 * m->sm_count))), dim3(kGenTile),
                                args, smem, st));
    m->launches++;
    return;
  }
  if (m->use_generic)
  {
    GenericKernelParams gp{};
    gp.weights = call.weights;
    gp.layers = m->d_glayers;
    gp.net = m->gplan.net;
    gp.cond = m->gplan.cond;
    gp.has_cond = m->gplan.has_cond ? 1 : 0;
    gp.state = call.state;
    gp.slots = call.slots;
    gp.state_stride = call.state_stride;
    gp.in = call.in;
    gp.out = call.out;
    gp.in_stride = call.in_stride;
    gp.out_stride = call.out_stride;
    gp.batch = batch;
    gp.n_frames = n_frames;
    gp.t_base = call.t_base;
    // (a bank: each model's blob with its two output scales behind the weights; its calls always carry a table)
    const bool bank = m->is_bank;
    gp.n_weight_floats = bank ? (int)m->weight_stride : (int)((m->n_weight_floats + 3) & ~(size_t)3);
    gp.weight_stride = call.weight_stride;
    gp.scale_off = (int)m->gplan.weights.size();
    const size_t wbytes = (size_t)gp.n_weight_floats * sizeof(float);
    const int grid_g = std::min(batch, 16 * m->sm_count);
    if (wbytes <= 200 * 1024)
    {
      auto kern = bank ? wavenet_generic_kernel<true, true, true>
                       : (call.slots ? wavenet_generic_kernel<true, true> : wavenet_generic_kernel<true>);
      ensure_max_dynamic_smem(reinterpret_cast<const void*>(kern), m->device, 200 * 1024);
      kern<<<grid_g, kGenTile, wbytes, st>>>(gp);
    }
    else
      (bank ? wavenet_generic_kernel<false, true, true>
            : (call.slots ? wavenet_generic_kernel<false, true> : wavenet_generic_kernel<false>))<<<grid_g, kGenTile, 0, st>>>(gp);
    CUDA_CHECK(cudaGetLastError());
    m->launches++;
    return;
  }
  const WaveNetPlan& plan = m->plan;
  WaveNetKernelParams kp{};
  kp.weights = call.weights;
  kp.n_weight_floats = (int)plan.blob.size();
  kp.state = call.state;
  kp.state_stride = call.state_stride;
  kp.slots = call.slots;
  kp.in = call.in;
  kp.out = call.out;
  kp.in_stride = call.in_stride;
  kp.out_stride = call.out_stride;
  kp.batch = batch;
  kp.n_frames = n_frames;
  kp.t_base = call.t_base;
  kp.head_scale = plan.head_scale;
  kp.weight_stride = call.weight_stride;
  kp.head_scales = m->d_head_scales; // (a bank's calls always carry a table: prefix_needs_table)
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
      launch_wavenet_lat(m, jp, st);
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
      void* args[] = {&jp};
      const int grid_s = std::max(1, std::min((batch + sv.q - 1) / sv.q, sv.ctas_per_sm * m->sm_count));
      CUDA_CHECK(cudaLaunchKernel((const void*)sv.kernel, dim3(grid_s), dim3(sv.fq * sv.q), args, sv.smem, st));
      m->launches++;
      return;
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
    launch_wavenet_spec(m, jp, st);
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
void setup_lstm_spec_kernel(nam_b200_model* m)
{
  if (!jit_wanted(m))
    return;
  const SpecBuild b = build_lstm_spec_kernel(m->spec);
  std::string why = b.ok ? m->spec_lib.load(b.cubin) : b.why_not;
  const char* const names[4] = {"lstm_spec_kernel_exact", "lstm_spec_kernel_fast", "lstm_spec_gates_kernel_exact",
                                "lstm_spec_gates_kernel_fast"};
  cudaKernel_t* const kernels[4] = {&m->lstm_spec_kernels[0], &m->lstm_spec_kernels[1], &m->lstm_gate_kernels[0],
                                    &m->lstm_gate_kernels[1]};
  for (int i = 0; i < 4 && why.empty(); i++)
    why = m->spec_lib.kernel(kernels[i], names[i]);
  if (!why.empty())
    return jit_unavailable(m, why, b.ok);
  m->spec_state = 1;
  m->spec_note = jit_loaded_note(b);
}

// ---- the general kernel compiled for this model (wavenet_generic_spec.cuh): same policy as the fused family's -------------
void setup_generic_spec_kernel(nam_b200_model* m)
{
  if (!jit_wanted(m) || m->opts.kernel_geometry == 4)
    return;
  const SpecBuild b = build_generic_spec_kernel(m->gplan);
  std::string why = b.why_not;
  if (b.ok)
  {
    std::string err = m->spec_lib.load(b.cubin);
    if (err.empty())
      err = m->spec_lib.kernel(&m->gen_spec_kernel, "wavenet_generic_spec_kernel");
    if (!err.empty())
      why = "loading the specialised general kernel failed: " + err;
  }
  if (!why.empty())
    return jit_unavailable(m, why, b.ok);
  m->spec_state = 1;
  m->spec_note = "general kernel, " + jit_loaded_note(b);
}

// A general-family bank: the general kernel compiled for the bank's shape (no weights in its code; each stream's blob is staged
// in shared memory), under the handle's jit policy.  Called once the bank's blobs are in place (setup_bank).
void setup_generic_bank_kernel(nam_b200_model* m)
{
  if (!jit_wanted(m) || m->opts.kernel_geometry == 4)
    return;
  const SpecBuild b = build_generic_spec_kernel(m->gplan, true);
  std::string why = b.why_not;
  if (b.ok)
  {
    std::string err = m->spec_lib.load(b.cubin);
    if (err.empty())
      err = m->spec_lib.kernel(&m->gen_spec_kernel, "wavenet_generic_spec_kernel", (size_t)m->weight_stride * sizeof(float),
                               kGenTile, &m->spec_ctas_per_sm);
    if (err.empty() && m->spec_ctas_per_sm < 1)
      err = "the shape-compiled general kernel does not fit on an SM";
    if (!err.empty())
      why = "loading the shape-compiled general kernel failed: " + err;
  }
  if (!why.empty())
    return jit_unavailable(m, "model bank of up to " + std::to_string(m->bank_capacity) + " models: " + why, b.ok);
  m->spec_state = 1;
  m->spec_note = "model bank of up to " + std::to_string(m->bank_capacity) + " models: the general kernel compiled for the bank's shape, "
                 + jit_loaded_note(b);
}

// (call.state: the handle's d_state, or the scratch rows nam_b200_reset_streams prewarms a gathered subset of streams in)
void launch_lstm(nam_b200_model* m, const JitParams& call, cudaStream_t st)
{
  const int batch = call.batch;
  if (m->spec_state == 1)
  {
    JitParams jp = call;
    void* args[] = {&jp};
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
  kp.weights = call.weights;
  kp.n_weight_floats = (int)m->n_weight_floats;
  kp.state = call.state;
  kp.state_stride = (int)call.state_stride;
  kp.in = call.in;
  kp.out = call.out;
  kp.in_stride = call.in_stride;
  kp.out_stride = call.out_stride;
  kp.batch = batch;
  kp.n_frames = call.n_frames;
  kp.num_layers = ls.num_layers;
  kp.input_size = ls.input_size;
  kp.hidden = ls.hidden;
  kp.fast_tanh = m->fast_tanh_runtime;
  kp.in_ch = m->spec.in_channels;
  kp.out_ch = m->spec.out_channels;
  kp.slots = call.slots;
  // a model bank: the BANK instantiations, which read each position's model from the table (whose host copy is
  // m->h_slots[0, batch)); the kernel family is the one an ordinary handle of the same shape gets
  const bool bank = m->is_bank;
  kp.weight_stride = call.weight_stride;
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
    const size_t io_floats = (size_t)2 * spc * (kLstmGroupChunk + 1);
    const size_t smem_g = (w_floats + H + 1 + io_floats) * sizeof(float);
    if (smem_g <= 227 * 1024)
    {
      const int grid_g = (batch + spc - 1) / spc;
      if (bank)
      {
        const void* kern = G == 4 ? (const void*)lstm_group_kernel<4, true>
                         : G == 8 ? (const void*)lstm_group_kernel<8, true>
                         : G == 16 ? (const void*)lstm_group_kernel<16, true> : (const void*)lstm_group_kernel<32, true>;
        // model copies: the most distinct models any CTA of this launch holds, capped by what fits beside the I/O tiles
        // and the kernel's static table of the CTA's models
        cudaFuncAttributes fa{};
        CUDA_CHECK(cudaFuncGetAttributes(&fa, kern));
        const size_t budget = 227 * 1024 - fa.sharedSizeBytes, copy_floats = w_floats + H + 1;
        const int fit = (int)std::min<size_t>((budget / sizeof(float) - io_floats) / copy_floats, (size_t)spc);
        if (fit < 1)
          throw std::runtime_error("LSTM bank: one model's weights do not fit in shared memory beside the bank's model table");
        kp.bank_copies = 1;
        for (int b0 = 0; b0 < batch && kp.bank_copies < fit; b0 += spc)
        {
          int seen[kLstmGroupThreads / 4], n = 0;
          for (int b = b0; b < std::min(batch, b0 + spc); b++)
          {
            const int k = m->h_slots[(size_t)b].model;
            if (std::find(seen, seen + n, k) == seen + n)
              seen[n++] = k;
          }
          kp.bank_copies = std::min(std::max(kp.bank_copies, n), fit);
        }
        ensure_max_dynamic_smem(kern, m->device, (int)budget);
        void* args[] = {&kp};
        CUDA_CHECK(cudaLaunchKernel(kern, dim3(grid_g), dim3(kLstmGroupThreads), args,
                                    (kp.bank_copies * copy_floats + io_floats) * sizeof(float), st));
        m->launches++;
        return;
      }
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
  const int grid = (batch + kLstmThreads - 1) / kLstmThreads;
  if (bank)
  {
    // (the kernel's static table of the CTA's models comes out of the same 227 KB)
    const void* kern = reinterpret_cast<const void*>(lstm_kernel<true>);
    cudaFuncAttributes fa{};
    CUDA_CHECK(cudaFuncGetAttributes(&fa, kern));
    const size_t budget = 227 * 1024 - fa.sharedSizeBytes;
    if (smem > budget)
      throw std::runtime_error("LSTM bank: one model's weights and state tiles do not fit in shared memory beside the bank's "
                               "model table");
    ensure_max_dynamic_smem(kern, m->device, (int)budget);
    lstm_kernel<true><<<grid, kLstmThreads, smem, st>>>(kp);
    CUDA_CHECK(cudaGetLastError());
    m->launches++;
    return;
  }
  ensure_max_dynamic_smem(reinterpret_cast<const void*>(lstm_kernel<false>), m->device, 227 * 1024);
  if (smem > 227 * 1024)
    throw std::runtime_error("LSTM too large for the shared-memory resident kernel");
  lstm_kernel<false><<<grid, kLstmThreads, smem, st>>>(kp);
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
}

// `slots` (with m->h_slots, its host copy): each listed stream reads the buffer its history is in and the update writes the
// other one -- no global swap, so streams left out keep theirs
void launch_linear(nam_b200_model* m, const JitParams& call, cudaStream_t st)
{
  const LinearSpec& li = m->spec.linear;
  const int batch = call.batch;
  const StreamRef* const slots = call.slots;
  LinearKernelParams kp{};
  kp.impulse = call.weights;
  kp.rf = li.receptive_field;
  kp.bias = li.bias_value;
  kp.state = call.state;
  kp.state_stride = (int)call.state_stride;
  kp.in = call.in;
  kp.out = call.out;
  kp.in_stride = call.in_stride;
  kp.out_stride = call.out_stride;
  kp.batch = batch;
  kp.n_frames = call.n_frames;
  kp.slots = slots;
  kp.state_alt = m->d_state_tmp;
  const size_t smem = (((size_t)li.receptive_field + 3) & ~(size_t)3) * 4 + ((size_t)li.receptive_field - 1 + kLinThreads) * 4;
  ensure_max_dynamic_smem(reinterpret_cast<const void*>(linear_kernel), m->device, 227 * 1024);
  if (smem > 227 * 1024)
    throw std::runtime_error("Linear receptive field too long for the direct-form kernel");
  if (batch > 65535)
    throw std::runtime_error("Linear: more than 65535 streams per call (grid.y); split the batch");
  dim3 grid((call.n_frames + kLinThreads - 1) / kLinThreads, batch);
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
    if (slots)
    {
      for (int b = 0; b < batch; b++)
        if (m->h_slots[(size_t)b].frames > 0) // (a stream that ran no frames stays on its side)
          m->stream_flips[(size_t)m->h_slots[(size_t)b].stream]++; // (only the parity against lin_flips matters)
      return;
    }
    std::swap(m->d_state, m->d_state_tmp);
    // streams [batch, max_batch) keep their history in the buffer they were last written to
    m->lin_flips++;
    for (int b = 0; b < batch; b++)
      m->stream_flips[(size_t)b] = m->lin_flips;
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

void launch_convnet(nam_b200_model* m, const JitParams& call, cudaStream_t st)
{
  ConvNetKernelParams kp{};
  kp.weights = call.weights;
  kp.net = m->gplan.convnet;
  kp.state = call.state;
  kp.state_stride = call.state_stride;
  kp.in = call.in;
  kp.out = call.out;
  kp.in_stride = call.in_stride;
  kp.out_stride = call.out_stride;
  kp.batch = call.batch;
  kp.n_frames = call.n_frames;
  kp.t_base = call.t_base;
  kp.n_weight_floats = (int)((m->n_weight_floats + 3) & ~(size_t)3);
  kp.slots = call.slots;
  kp.weight_stride = call.weight_stride; // (a bank: its calls always carry a table)
  const bool bank = m->is_bank;
  const size_t wbytes = (size_t)kp.n_weight_floats * sizeof(float);
  const int grid = std::min(call.batch, 16 * m->sm_count);
  if (wbytes <= 200 * 1024)
  {
    auto kern = bank ? convnet_kernel<true, true, true> : (call.slots ? convnet_kernel<true, true> : convnet_kernel<true>);
    ensure_max_dynamic_smem(reinterpret_cast<const void*>(kern), m->device, 200 * 1024);
    kern<<<grid, kGenTile, wbytes, st>>>(kp);
  }
  else
    (bank ? convnet_kernel<false, true, true>
          : (call.slots ? convnet_kernel<false, true> : convnet_kernel<false>))<<<grid, kGenTile, 0, st>>>(kp);
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
}

// One call of the handle's kernel on `st`, described as jit_params() describes it
void launch(nam_b200_model* m, const JitParams& call, cudaStream_t st)
{
  switch (m->spec.arch)
  {
    case Arch::WaveNet: return launch_wavenet(m, call, st);
    case Arch::LSTM: return launch_lstm(m, call, st);
    case Arch::Linear: return launch_linear(m, call, st);
    case Arch::ConvNet: return launch_convnet(m, call, st);
    default: throw std::runtime_error("no kernel for this architecture");
  }
}

// ---- per-stream clocks and slot tables ----------------------------------------------------------------------------------
// Does where stream s's history ends matter to the next call over it?  WaveNet / ConvNet rings are addressed by the clock;
// Linear's flat history has no clock but lives in one buffer of a double buffer; an LSTM's h, c are just its state.
bool phase_matters(const nam_b200_model* m)
{
  return m->spec.arch == Arch::WaveNet || m->spec.arch == Arch::ConvNet
         || (m->spec.arch == Arch::Linear && m->spec.linear.receptive_field > 1);
}
bool in_phase(const nam_b200_model* m, size_t s)
{
  if (m->spec.arch == Arch::Linear)
    return m->spec.linear.receptive_field <= 1 || ((m->lin_flips - m->stream_flips[s]) & 1u) == 0;
  return !phase_matters(m) || m->stream_clock[s] == m->t_base;
}
void recount_phase(nam_b200_model* m)
{
  int n = 0;
  for (size_t s = 0; s < m->stream_clock.size(); s++)
    n += in_phase(m, s) ? 0 : 1;
  m->n_out_of_phase = n;
}
// Must a contiguous call over streams [0, batch) carry an identity slot table (one of them sat out calls, or the handle is a
// model bank, whose table carries each position's model)?  O(1) while every stream is in phase (a handle that always runs
// all its streams).
bool prefix_needs_table(const nam_b200_model* m, int batch)
{
  if (m->is_bank)
    return true;
  if (m->n_out_of_phase == 0)
    return false;
  for (int b = 0; b < batch; b++)
    if (!in_phase(m, (size_t)b))
      return true;
  return false;
}

// The call's slot table (streams[i], or i when streams == nullptr; counts[i] frames, or n_frames each when counts ==
// nullptr) -> m->h_slots -> the device table, ordered on `st` before the launches that read it.  The host copy is
// pageable: cudaMemcpyAsync stages it before returning, so the next call may rebuild it at once.  The device table waits
// for the previous table call's launches (slots_free).
const StreamRef* push_slots(nam_b200_model* m, int n, cudaStream_t st)
{
  if (m->slots_used)
    CUDA_CHECK(cudaStreamWaitEvent(st, m->slots_free, 0));
  CUDA_CHECK(cudaMemcpyAsync(m->d_slots, m->h_slots.data(), (size_t)n * sizeof(StreamRef), cudaMemcpyHostToDevice, st));
  return m->d_slots;
}
// After the launches that read the device table: the next push_slots waits for them
void release_slots(nam_b200_model* m, cudaStream_t st)
{
  CUDA_CHECK(cudaEventRecord(m->slots_free, st));
  m->slots_used = true;
}
const StreamRef* upload_slots(nam_b200_model* m, const int32_t* streams, int n, int n_frames, const int32_t* counts,
                              cudaStream_t st)
{
  const bool linear = m->spec.arch == Arch::Linear;
  for (int i = 0; i < n; i++)
  {
    const int32_t s = streams ? streams[i] : i;
    // (Linear: the buffer the history is in; every other architecture: the stream's model, 0 outside a bank)
    m->h_slots[(size_t)i] = StreamRef{s, m->stream_clock[(size_t)s],
                                      linear ? ((m->lin_flips - m->stream_flips[(size_t)s]) & 1u ? 1 : 0) : m->stream_model[(size_t)s],
                                      counts ? counts[i] : n_frames};
  }
  return push_slots(m, n, st);
}

// After the launches of a table call on `st`: each listed stream's history moved on by its own count, the handle's clock
// by the call's n_frames (the longest count)
void finish_table_call(nam_b200_model* m, int n, int n_frames, cudaStream_t st)
{
  release_slots(m, st);
  m->t_base += (uint32_t)n_frames;
  for (int i = 0; i < n; i++)
    m->stream_clock[(size_t)m->h_slots[(size_t)i].stream] += (uint32_t)m->h_slots[(size_t)i].frames;
  m->streams_identical = false;
  recount_phase(m);
}

// After a contiguous call without a table over [0, batch): those streams end at the new t_base, the others fell behind
void finish_contiguous_call(nam_b200_model* m, int batch, int n_frames)
{
  m->t_base += (uint32_t)n_frames;
  std::fill(m->stream_clock.begin(), m->stream_clock.begin() + batch, m->t_base);
  m->n_out_of_phase = phase_matters(m) ? m->opts.max_batch - batch : 0;
  m->streams_identical = false; // (prewarm() restores the flag: it feeds every stream the same zeros)
}

// Run the hot path on device buffers and advance the stream clocks.  `streams` (n = batch entries): the call's positions
// run these streams, each from its own clock.  nullptr: streams [0, batch) -- launched without a table while all of them
// are in phase, else with the identity table (a stream that sat out calls continues from its own clock).  `counts`
// (with `streams`): position i runs counts[i] <= n_frames frames; n_frames stays the buffers' frame pitch.
void run_device(nam_b200_model* m, const float* d_in, float* d_out, int batch, int n_frames, long in_stride,
                long out_stride, cudaStream_t st, const int32_t* streams = nullptr, const int32_t* counts = nullptr)
{
  const bool table = streams != nullptr || prefix_needs_table(m, batch);
  const StreamRef* slots = table ? upload_slots(m, streams, batch, n_frames, counts, st) : nullptr;
  launch(m, jit_params(m, m->d_state, d_in, d_out, in_stride, out_stride, batch, n_frames, slots), st);
  if (table)
    finish_table_call(m, batch, n_frames, st);
  else
    finish_contiguous_call(m, batch, n_frames);
}

// every stream's history ends at the handle's clock (init_state, prewarm)
void set_all_clocks(nam_b200_model* m)
{
  std::fill(m->stream_clock.begin(), m->stream_clock.end(), m->t_base);
  std::fill(m->stream_flips.begin(), m->stream_flips.end(), m->lin_flips);
  m->n_out_of_phase = 0;
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

// ---- sample-rate conversion (options.resample; resample.h, resample.cuh) ----------------------------------------------
// host frames a process call may carry: maxBufferSize of the last reset
int call_max_frames(const nam_b200_model* m)
{
  return m->rs.active ? m->rs.host_max_frames : m->max_frames;
}
// frames per stream of the host staging buffers: host calls and the model's own calls (prewarm) both pass through them
int staging_frames(const nam_b200_model* m)
{
  return std::max(m->max_frames, call_max_frames(m));
}

// dynamic shared memory of one conversion launch: the phase table and the input window of `tile` outputs
size_t rs_smem_bytes(int T, int A, int B, int tile)
{
  return 4 * ((size_t)T * B + (size_t)(tile - 1) * A / B + T + 2);
}

void free_resampler(nam_b200_model* m)
{
  auto& r = m->rs;
  for (float** p : {&r.d_taps, &r.d_hist, &r.d_x, &r.d_z})
  {
    if (*p)
      cudaFree(*p);
    *p = nullptr;
  }
  if (r.d_pos)
    cudaFree(r.d_pos);
  r.d_pos = nullptr;
  r.active = false;
}

// The conversion nam_b200_reset(host_rate) needs: *d and true, or false when none is (resample = 0, equal rates).
// Returns the refusal ("" when fine) -- checked before reset changes anything.
std::string resampler_for(const nam_b200_model* m, double host_rate, ResamplerDesign* d, bool* needed)
{
  *needed = m->opts.resample != 0 && host_rate != m->spec.sample_rate;
  std::string why;
  if (!*needed)
    return why;
  if (design_resampler(host_rate, m->spec.sample_rate, d, &why))
  {
    int optin = 0;
    CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, m->device));
    const size_t smem = std::max(rs_smem_bytes(d->taps_up, d->M, d->L, kRsMaxThreads), rs_smem_bytes(d->taps_dn, d->L, d->M, kRsMaxThreads));
    if (smem > (size_t)optin)
      why = "resample: host rate " + std::to_string((long long)host_rate) + " Hz, model rate " + std::to_string((long long)m->spec.sample_rate)
            + " Hz: the phase tables need " + std::to_string(smem) + " bytes of shared memory, more than the device's "
            + std::to_string(optin);
  }
  return why;
}

// nam_b200_reset's part: every stream's conversion state zero, h = 0; m->max_frames becomes the model's maxBufferSize
void setup_resampler(nam_b200_model* m, bool needed, const ResamplerDesign& d, int max_frames)
{
  free_resampler(m);
  m->max_frames = max_frames;
  if (!needed)
    return;
  auto& r = m->rs;
  const int ci = m->spec.in_channels, co = m->spec.out_channels, nb = m->opts.max_batch;
  r.design = d;
  r.H_up = d.taps_up;
  r.H_dn = d.taps_dn;
  r.rs_stride = (ci * r.H_up + co * r.H_dn + 3) & ~3;
  r.host_max_frames = max_frames;
  m->max_frames = (int)(((int64_t)max_frames * d.L + d.M - 1) / d.M);
  std::vector<float> taps = resampler_phase_table(d.g_up, d.L, d.taps_up);
  const std::vector<float> dn = resampler_phase_table(d.g_dn, d.M, d.taps_dn);
  taps.insert(taps.end(), dn.begin(), dn.end());
  CUDA_CHECK(cudaMalloc(&r.d_taps, taps.size() * sizeof(float)));
  CUDA_CHECK(cudaMemcpy(r.d_taps, taps.data(), taps.size() * sizeof(float), cudaMemcpyHostToDevice));
  const size_t hist = (size_t)(nb + 1) * r.rs_stride;
  CUDA_CHECK(cudaMalloc(&r.d_hist, hist * sizeof(float)));
  CUDA_CHECK(cudaMemsetAsync(r.d_hist, 0, hist * sizeof(float), m->stream));
  CUDA_CHECK(cudaMalloc(&r.d_x, (size_t)nb * ci * m->max_frames * sizeof(float)));
  CUDA_CHECK(cudaMalloc(&r.d_z, (size_t)nb * co * m->max_frames * sizeof(float)));
  CUDA_CHECK(cudaMalloc(&r.d_pos, (size_t)nb * sizeof(RsPos)));
  if (!r.pos_free)
    CUDA_CHECK(cudaEventCreateWithFlags(&r.pos_free, cudaEventDisableTiming));
  r.pos_used = false;
  r.phase.assign((size_t)nb, 0u);
  r.h_pos.assign((size_t)nb, RsPos{0, 0, 0, 0});
  int optin = 0;
  CUDA_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, m->device));
  ensure_max_dynamic_smem((const void*)resample_kernel<true>, m->device, optin);
  ensure_max_dynamic_smem((const void*)resample_kernel<false>, m->device, optin);
  r.active = true;
}

// One direction over the call's positions (m->rs.d_pos): up = host -> model.  n_out_max: the longest output row.
void launch_resample(nam_b200_model* m, bool up, const float* in, long in_stride, int in_pitch, float* out, long out_stride,
                     int out_pitch, int n_pos, int n_out_max, cudaStream_t st)
{
  if (n_out_max == 0)
    return;
  const auto& r = m->rs;
  const ResamplerDesign& d = r.design;
  ResampleParams p{};
  p.T = up ? d.taps_up : d.taps_dn;
  p.A = up ? d.M : d.L;
  p.B = up ? d.L : d.M;
  p.taps = r.d_taps + (up ? 0 : (size_t)d.taps_up * d.L);
  p.pos = r.d_pos;
  p.n_pos = n_pos;
  p.in = in;
  p.in_stride = in_stride;
  p.in_pitch = in_pitch;
  p.out = out;
  p.out_stride = out_stride;
  p.out_pitch = out_pitch;
  p.hist = r.d_hist;
  p.hist_stride = r.rs_stride;
  p.hist_off = up ? 0 : m->spec.in_channels * r.H_up;
  p.H = up ? r.H_up : r.H_dn;
  const int tile = std::min(kRsMaxThreads, (n_out_max + 31) & ~31);
  const int tiles = (n_out_max + tile - 1) / tile;
  const int ch = up ? m->spec.in_channels : m->spec.out_channels;
  // positions per CTA: about four CTAs per SM in all, so that each stages the phase table once for many rows
  p.group = (int)std::max<long>(1, (long)n_pos * tiles * ch / (4L * std::max(m->sm_count, 1)));
  const dim3 grid((unsigned)((n_pos + p.group - 1) / p.group), (unsigned)tiles, (unsigned)ch);
  const size_t smem = rs_smem_bytes(p.T, p.A, p.B, tile);
  if (up)
    resample_kernel<true><<<grid, tile, smem, st>>>(p);
  else
    resample_kernel<false><<<grid, tile, smem, st>>>(p);
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
}

// run_device for the process entries: on a converting handle, host -> model into rs.d_x, the model's launch over it (per
// position its own count of model frames), model -> host into d_out, then the histories; otherwise run_device itself.
// `n_frames` is the call's host frame pitch (the longest row of a ragged call).
void run_call(nam_b200_model* m, const float* d_in, float* d_out, int batch, int n_frames, long in_stride, long out_stride,
              cudaStream_t st, const int32_t* streams = nullptr, const int32_t* counts = nullptr)
{
  auto& r = m->rs;
  if (!r.active)
    return run_device(m, d_in, d_out, batch, n_frames, in_stride, out_stride, st, streams, counts);
  const int64_t L = r.design.L, M = r.design.M;
  int m_max = 0;
  bool equal = true;
  for (int i = 0; i < batch; i++)
  {
    const int s = streams ? streams[i] : i;
    const int n = counts ? counts[i] : n_frames;
    const int64_t ph = r.phase[(size_t)s];
    const int mi = (int)(((ph + n) * L + M - 1) / M - (ph * L + M - 1) / M);
    r.h_pos[(size_t)i] = RsPos{s, (int)((M - (ph * L) % M) % M), n, mi};
    m_max = std::max(m_max, mi);
    equal = equal && mi == r.h_pos[0].m;
  }
  if (r.pos_used)
    CUDA_CHECK(cudaStreamWaitEvent(st, r.pos_free, 0));
  CUDA_CHECK(cudaMemcpyAsync(r.d_pos, r.h_pos.data(), (size_t)batch * sizeof(RsPos), cudaMemcpyHostToDevice, st));
  const int ci = m->spec.in_channels, co = m->spec.out_channels;
  launch_resample(m, true, d_in, in_stride, n_frames, r.d_x, (long)ci * m_max, m_max, batch, m_max, st);
  if (m_max > 0)
  {
    if (!streams && equal)
      run_device(m, r.d_x, r.d_z, batch, m_max, (long)ci * m_max, (long)co * m_max, st);
    else
    {
      std::vector<int32_t> ids((size_t)batch), cnt((size_t)batch);
      for (int i = 0; i < batch; i++)
      {
        ids[(size_t)i] = r.h_pos[(size_t)i].stream;
        cnt[(size_t)i] = r.h_pos[(size_t)i].m;
      }
      run_device(m, r.d_x, r.d_z, batch, m_max, (long)ci * m_max, (long)co * m_max, st, ids.data(), equal ? nullptr : cnt.data());
    }
  }
  launch_resample(m, false, r.d_z, (long)co * m_max, m_max, d_out, out_stride, n_frames, batch, n_frames, st);
  ResampleHistoryParams hp{};
  hp.pos = r.d_pos;
  hp.in_channels = ci;
  hp.x = d_in;
  hp.x_stride = in_stride;
  hp.x_pitch = n_frames;
  hp.z = r.d_z;
  hp.z_stride = (long)co * m_max;
  hp.z_pitch = m_max;
  hp.hist = r.d_hist;
  hp.hist_stride = r.rs_stride;
  hp.H_up = r.H_up;
  hp.H_dn = r.H_dn;
  resample_history_kernel<<<dim3((unsigned)batch, (unsigned)(ci + co)), kRsHistThreads, 0, st>>>(hp);
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
  CUDA_CHECK(cudaEventRecord(r.pos_free, st));
  r.pos_used = true;
  for (int i = 0; i < batch; i++)
  {
    const RsPos& p = r.h_pos[(size_t)i];
    r.phase[(size_t)p.stream] = (uint32_t)((r.phase[(size_t)p.stream] + (uint32_t)p.n) % (uint32_t)M);
  }
}

// Zero the state, set the trained initial state where the architecture has one.
// state rows of the handle: one per stream, plus a bank's model rows
int state_rows(const nam_b200_model* m)
{
  return m->opts.max_batch + (m->is_bank ? m->bank_capacity : 0);
}

// model k's document (a bank's; model 0 of an ordinary handle is its own)
const ModelSpec& model_spec(const nam_b200_model* m, int k)
{
  return m->is_bank ? m->bank_specs[(size_t)k] : m->spec;
}

// an LSTM's trained initial state (lstm.cpp:24-28) as one state row: per layer h0[H] | c0[H]
void lstm_initial_row(const ModelSpec& s, float* row)
{
  const int H = s.lstm.hidden;
  for (int l = 0; l < s.lstm.num_layers; l++)
  {
    std::copy(s.lstm.cells[l].h0.begin(), s.lstm.cells[l].h0.end(), row + (size_t)l * 2 * H);
    std::copy(s.lstm.cells[l].c0.begin(), s.lstm.cells[l].c0.end(), row + (size_t)l * 2 * H + H);
  }
}

// rows [r0, r0 + n) of `state` take the h0 / c0 of models[i] (a bank's model rows; the rows of a reset_streams call)
void write_lstm_initial_rows(nam_b200_model* m, float* state, size_t r0, const std::vector<int32_t>& models)
{
  const size_t stride = (size_t)m->state_stride;
  std::vector<float> h(models.size() * stride, 0.0f);
  for (size_t i = 0; i < models.size(); i++)
    lstm_initial_row(model_spec(m, models[i]), h.data() + i * stride);
  // (h is pageable: the copy stages it before returning)
  CUDA_CHECK(cudaMemcpyAsync(state + r0 * stride, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice, m->stream));
}

void init_state(nam_b200_model* m)
{
  const size_t total = (size_t)m->state_stride * state_rows(m);
  m->fresh_clock = 0;
  CUDA_CHECK(cudaMemsetAsync(m->d_state, 0, total * sizeof(float), m->stream));
  if (m->spec.arch == Arch::LSTM)
  {
    // h0 / c0 are trained parameters (lstm.cpp:24-28): every stream starts from its model's, as every reference DSP object
    // does (prewarm_on_reset = 0 runs no prewarm to broadcast them); a bank's model row k from model k's
    std::vector<int32_t> models(m->stream_model);
    for (int k = 0; k < (m->is_bank ? m->bank_size : 0); k++)
      models.push_back(k);
    write_lstm_initial_rows(m, m->d_state, 0, models);
  }
  if (m->spec.arch == Arch::Linear && m->d_state_tmp)
    CUDA_CHECK(cudaMemsetAsync(m->d_state_tmp, 0, total * sizeof(float), m->stream));
  m->t_base = 0;
  set_all_clocks(m);
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

// DSP::prewarm's loop (dsp.cpp:67-101): zeros in max_frames blocks until >= prewarm_samples.  The staging is sized for
// `rows` streams and the input of the first n zeroed; block(call) runs each block, `call` being n positions of zeros on
// the handle's state rows without a table.  Nothing happens without prewarm samples.
template <typename F>
void prewarm_blocks(nam_b200_model* m, int n, int rows, const F& block)
{
  const int ps = m->spec.prewarm_samples;
  if (ps <= 0)
    return;
  const int bs = std::max(m->max_frames, 1);
  const size_t ci = (size_t)m->spec.in_channels, co = (size_t)m->spec.out_channels;
  ensure_staging(m, (size_t)rows * bs * std::max(ci, co));
  CUDA_CHECK(cudaMemsetAsync(m->d_in, 0, (size_t)n * bs * ci * sizeof(float), m->stream));
  for (int done = 0; done < ps; done += bs)
    block(jit_params(m, m->d_state, m->d_in, m->d_out, (long)(bs * ci), (long)(bs * co), n, bs, nullptr));
}

// `call` with the first n entries of m->h_slots as its table
void launch_with_table(nam_b200_model* m, JitParams call, int n, cudaStream_t st)
{
  call.slots = push_slots(m, n, st);
  launch(m, call, st);
  release_slots(m, st);
}

// DSP::prewarm: done once on stream 0 (every stream would compute the identical state) and broadcast.
void prewarm(nam_b200_model* m)
{
  if (m->spec.prewarm_samples <= 0)
    return;
  // DSP::prewarm continues from the instance's CURRENT state (dsp.cpp:67-101).  Straight after init_state every stream
  // would compute the same thing: stream 0 runs, its state is broadcast.  Once the streams have seen different audio
  // (a standalone nam_b200_prewarm, or a Reset of an LSTM, which keeps its running state) all of them are prewarmed.
  // (a bank's streams run different models: nam_b200_reset prewarms it through prewarm_bank or prewarm_lstm_bank, a
  // standalone prewarm runs every stream with its own model)
  const bool identical = m->streams_identical && !m->is_bank;
  prewarm_blocks(m, identical ? 1 : m->opts.max_batch, m->opts.max_batch, [&](const JitParams& c) {
    run_device(m, c.in, c.out, c.batch, c.n_frames, c.in_stride, c.out_stride, m->stream);
  });
  m->streams_identical = identical; // zeros into identical streams keep them identical
  if (identical)
  {
    // every stream now holds stream 0's state, in d_state, ending where stream 0's does
    broadcast_state(m);
    if (m->spec.arch == Arch::Linear && m->d_state_tmp)
      CUDA_CHECK(cudaMemcpyAsync(m->d_state_tmp, m->d_state, (size_t)m->state_stride * m->opts.max_batch * sizeof(float),
                                 cudaMemcpyDeviceToDevice, m->stream));
    set_all_clocks(m);
  }
  // (otherwise every stream ran from its own clock -- with the identity table when one of them sat out calls -- and
  // run_device left each clock and Linear buffer where that stream's history now ends: a stream that was behind stays behind)
  CUDA_CHECK(cudaStreamSynchronize(m->stream));
}

// ---- per-stream state records (stream_state.h / .cuh) ------------------------------------------------------------------
// The handle's descriptor table, built once at creation.  A layout the record cannot describe (an internal mismatch) leaves
// the handle working and only the stream-state calls refused, with the reason (nam_b200_model::state_error).
// payload floats the conversion appends to a record (resample_in, resample_out, resample_phase), and its header word 3
long rs_record_floats(const nam_b200_model* m)
{
  const auto& r = m->rs;
  return r.active ? (long)m->spec.in_channels * r.H_up + (long)m->spec.out_channels * r.H_dn + 1 : 0;
}
uint32_t rs_ratio(const nam_b200_model* m)
{
  return m->rs.active ? ((uint32_t)m->rs.design.L << 16 | (uint32_t)m->rs.design.M) : 0u;
}

size_t record_bytes(const nam_b200_model* m)
{
  return (size_t)kStateHeaderBytes + 4 * (size_t)(m->record_floats + rs_record_floats(m));
}

void setup_state_records(nam_b200_model* m)
{
  const bool gen = (m->spec.arch == Arch::WaveNet && m->use_generic) || m->spec.arch == Arch::ConvNet;
  const bool fused = m->spec.arch == Arch::WaveNet && !m->use_generic;
  m->state_descs = state_descs(m->spec, fused ? &m->plan : nullptr, gen ? &m->gplan : nullptr);
  m->record_floats = 0;
  for (const StateSegDesc& d : m->state_descs)
    m->record_floats += (long)d.lookback * d.cr;
  if (m->state_descs.empty()) // (a model without history: launches still write the record headers)
    m->state_descs.push_back(StateSegDesc{kSegFlat, 0, 1, 1, 0, 0, 0, 0});
  m->state_chunks = state_chunks(m->state_descs);
  if (m->state_chunks.empty())
    m->state_chunks.push_back(StateChunk{0, 0});
  m->record_header = state_record_header(m->spec, m->record_floats);
  CUDA_CHECK(cudaMalloc(&m->d_state_descs, m->state_descs.size() * sizeof(StateSegDesc)));
  CUDA_CHECK(cudaMemcpy(m->d_state_descs, m->state_descs.data(), m->state_descs.size() * sizeof(StateSegDesc), cudaMemcpyHostToDevice));
  CUDA_CHECK(cudaMalloc(&m->d_state_chunks, m->state_chunks.size() * sizeof(StateChunk)));
  CUDA_CHECK(cudaMemcpy(m->d_state_chunks, m->state_chunks.data(), m->state_chunks.size() * sizeof(StateChunk), cudaMemcpyHostToDevice));
  CUDA_CHECK(cudaMalloc(&m->d_fresh, record_bytes(m)));
}

void ensure_xfer(nam_b200_model* m, size_t bytes)
{
  if (bytes <= m->xfer_bytes)
    return;
  if (m->d_xfer)
    cudaFree(m->d_xfer);
  m->d_xfer = nullptr;
  m->xfer_bytes = 0;
  CUDA_CHECK(cudaMalloc(&m->d_xfer, bytes));
  m->xfer_bytes = bytes;
}

// stream list -> device (d_refs); ordered on `st` before the launch that reads it
const StreamRef* upload_refs(nam_b200_model* m, const std::vector<StreamRef>& refs, cudaStream_t st)
{
  if (refs.size() > m->refs_capacity)
  {
    if (m->d_refs)
      cudaFree(m->d_refs);
    m->d_refs = nullptr;
    m->refs_capacity = 0;
    CUDA_CHECK(cudaMalloc(&m->d_refs, refs.size() * sizeof(StreamRef)));
    m->refs_capacity = refs.size();
  }
  CUDA_CHECK(cudaMemcpyAsync(m->d_refs, refs.data(), refs.size() * sizeof(StreamRef), cudaMemcpyHostToDevice, st));
  return m->d_refs;
}

dim3 state_grid(const nam_b200_model* m, int n)
{
  return dim3((unsigned)m->state_chunks.size(), (unsigned)std::min(n, 65535));
}

// pack streams[0..n) at their own clocks into records dst + i * stride
void export_records(nam_b200_model* m, const int32_t* streams, int n, unsigned char* dst, long stride, cudaStream_t st)
{
  std::vector<StreamRef> refs((size_t)n);
  const bool linear = m->spec.arch == Arch::Linear;
  for (int i = 0; i < n; i++)
  {
    const size_t s = (size_t)streams[i];
    refs[(size_t)i] = StreamRef{streams[i], m->stream_clock[s],
                                linear ? ((m->lin_flips - m->stream_flips[s]) & 1u ? 1 : 0) : m->stream_model[s], 0};
  }
  StatePackParams p{};
  p.segs = m->d_state_descs;
  p.chunks = m->d_state_chunks;
  p.state = m->d_state;
  p.state_alt = m->d_state_tmp ? m->d_state_tmp : m->d_state;
  p.state_stride = m->state_stride;
  p.refs = upload_refs(m, refs, st);
  p.n = n;
  p.rec = dst;
  p.rec_stride = stride;
  std::memcpy(p.header, &m->record_header, sizeof p.header);
  p.headers = m->d_bank_headers; // (a bank: the header of each stream's model)
  state_pack_kernel<<<state_grid(m, n), kStateThreads, 0, st>>>(p);
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
}

// the streams' histories now end at the handle's clock, in the buffer the next call reads
void mark_written(nam_b200_model* m, const int32_t* streams, int n)
{
  for (int i = 0; i < n; i++)
  {
    m->stream_clock[(size_t)streams[i]] = m->t_base;
    m->stream_flips[(size_t)streams[i]] = m->lin_flips;
  }
  m->streams_identical = false; // (a later prewarm must not broadcast stream 0 over them)
  recount_phase(m);
}

// unpack records src + i * stride (stride 0: one record for all) into streams[0..n) at the handle's clock
void import_records(nam_b200_model* m, const int32_t* streams, int n, const unsigned char* src, long stride, cudaStream_t st)
{
  std::vector<StreamRef> refs((size_t)n);
  for (int i = 0; i < n; i++)
    refs[(size_t)i] = StreamRef{streams[i], m->t_base, 0, 0};
  StateUnpackParams p{};
  p.segs = m->d_state_descs;
  p.chunks = m->d_state_chunks;
  p.state = m->d_state;
  p.state_stride = m->state_stride;
  p.refs = upload_refs(m, refs, st);
  p.n = n;
  p.rec = src;
  p.rec_stride = stride;
  state_unpack_kernel<<<state_grid(m, n), kStateThreads, 0, st>>>(p);
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
  mark_written(m, streams, n);
}

// ---- the conversion's part of the per-stream state (a converting handle only) ------------------------------------------
ResampleRecordParams rs_record_params(nam_b200_model* m, const int32_t* streams, int n, const uint32_t* phases, unsigned char* rec,
                                      long stride, cudaStream_t st)
{
  std::vector<StreamRef> refs((size_t)n);
  for (int i = 0; i < n; i++)
    refs[(size_t)i] = StreamRef{streams[i], phases ? phases[i] : m->rs.phase[(size_t)streams[i]], 0, 0};
  ResampleRecordParams p{};
  p.hist = m->rs.d_hist;
  p.hist_stride = m->rs.rs_stride;
  p.in_channels = m->spec.in_channels;
  p.out_channels = m->spec.out_channels;
  p.H_up = m->rs.H_up;
  p.H_dn = m->rs.H_dn;
  p.refs = upload_refs(m, refs, st);
  p.n = n;
  p.rec = rec;
  p.rec_stride = stride;
  p.off = m->record_floats;
  p.ratio = rs_ratio(m);
  p.payload_floats = (uint64_t)(m->record_floats + rs_record_floats(m));
  return p;
}
dim3 rs_record_grid(const nam_b200_model* m, int n)
{
  return dim3((unsigned)((rs_record_floats(m) - 1 + 255) / 256), (unsigned)std::min(n, 65535)); // (>= 1 item: H >= 1)
}

// after export_records into the same records: the conversion's segments and the header's ratio and payload count
void rs_export(nam_b200_model* m, const int32_t* streams, int n, unsigned char* dst, long stride, cudaStream_t st)
{
  if (!m->rs.active)
    return;
  resample_pack_kernel<<<rs_record_grid(m, n), 256, 0, st>>>(rs_record_params(m, streams, n, nullptr, dst, stride, st));
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
}

// the records' conversion segments into the streams; phases[i] = record i's resample_phase, checked by the caller
void rs_import(nam_b200_model* m, const int32_t* streams, int n, const unsigned char* src, long stride, const uint32_t* phases,
               cudaStream_t st)
{
  if (!m->rs.active)
    return;
  resample_unpack_kernel<<<rs_record_grid(m, n), 256, 0, st>>>(
    rs_record_params(m, streams, n, phases, const_cast<unsigned char*>(src), stride, st));
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
  for (int i = 0; i < n; i++)
    m->rs.phase[(size_t)streams[i]] = phases[i];
}

// record i's resample_phase (a float at the end of its payload) -> phases[i]; refused unless an integer in [0, M)
int rs_record_phases(const nam_b200_model* m, const int32_t* streams, const float* values, int n, std::vector<uint32_t>* phases)
{
  phases->assign((size_t)n, 0u);
  for (int i = 0; i < n; i++)
  {
    const float v = values[i];
    if (!(v >= 0.0f && v < (float)m->rs.design.M && std::floor(v) == v))
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, "record " + std::to_string(i) + " (stream " + std::to_string(streams[i])
                                                   + "): resample_phase " + std::to_string(v) + " is not an integer in [0, M="
                                                   + std::to_string(m->rs.design.M) + ")");
    (*phases)[(size_t)i] = (uint32_t)v;
  }
  return NAM_B200_OK;
}

// reset_streams / assign_streams: zero histories (row max_batch), h = 0
void rs_zero(nam_b200_model* m, const int32_t* streams, int n, cudaStream_t st)
{
  if (!m->rs.active)
    return;
  std::vector<StreamRef> refs((size_t)2 * n);
  for (int i = 0; i < n; i++)
  {
    refs[(size_t)i] = StreamRef{m->opts.max_batch, 0, 0, 0};
    refs[(size_t)(n + i)] = StreamRef{streams[i], 0, 0, 0};
    m->rs.phase[(size_t)streams[i]] = 0;
  }
  const StreamRef* d_refs = upload_refs(m, refs, st);
  const long stride4 = m->rs.rs_stride / 4;
  const dim3 grid((unsigned)((stride4 + kStateThreads - 1) / kStateThreads), (unsigned)std::min(n, 65535));
  state_rows_kernel<<<grid, kStateThreads, 0, st>>>(reinterpret_cast<float4*>(m->rs.d_hist), reinterpret_cast<const float4*>(m->rs.d_hist),
                                                     stride4, d_refs + n, d_refs, n);
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
}

// copy_streams: dst[i] takes src[i]'s conversion state, through scratch (a swap works)
void rs_copy(nam_b200_model* m, const int32_t* src, const int32_t* dst, int n, cudaStream_t st)
{
  if (!m->rs.active)
    return;
  const long stride4 = m->rs.rs_stride / 4;
  ensure_xfer(m, (size_t)n * m->rs.rs_stride * sizeof(float));
  std::vector<StreamRef> refs((size_t)2 * n);
  std::vector<uint32_t> ph((size_t)n);
  for (int i = 0; i < n; i++)
  {
    refs[(size_t)i] = StreamRef{src[i], 0, 0, 0};
    refs[(size_t)(n + i)] = StreamRef{dst[i], 0, 0, 0};
    ph[(size_t)i] = m->rs.phase[(size_t)src[i]];
  }
  const StreamRef* d_refs = upload_refs(m, refs, st);
  float4* scratch = reinterpret_cast<float4*>(m->d_xfer);
  float4* hist = reinterpret_cast<float4*>(m->rs.d_hist);
  const dim3 grid((unsigned)((stride4 + kStateThreads - 1) / kStateThreads), (unsigned)std::min(n, 65535));
  state_rows_kernel<<<grid, kStateThreads, 0, st>>>(scratch, hist, stride4, nullptr, d_refs, n);
  state_rows_kernel<<<grid, kStateThreads, 0, st>>>(hist, scratch, stride4, d_refs + n, nullptr, n);
  CUDA_CHECK(cudaGetLastError());
  m->launches += 2;
  for (int i = 0; i < n; i++)
    m->rs.phase[(size_t)dst[i]] = ph[(size_t)i];
}

// whole state rows: dst[dst_refs[i].stream or i] = src[src_refs[i].stream or i]
void copy_rows(nam_b200_model* m, float* dst, const StreamRef* dst_refs, const float* src, const StreamRef* src_refs, int n,
               cudaStream_t st)
{
  const long stride4 = m->state_stride / 4;
  const dim3 grid((unsigned)((stride4 + kStateThreads - 1) / kStateThreads), (unsigned)std::min(n, 65535));
  state_rows_kernel<<<grid, kStateThreads, 0, st>>>(reinterpret_cast<float4*>(dst), reinterpret_cast<const float4*>(src), stride4,
                                                      dst_refs, src_refs, n);
  CUDA_CHECK(cudaGetLastError());
  m->launches++;
}

// nam_b200_reset for an LSTM keeps h, c and prewarms on top (fresh: from h0 / c0, like a new handle): the listed streams'
// rows are gathered into scratch, prewarmed there exactly like prewarm() (zeros in max_frames blocks), scattered back.  A
// bank's launches carry a table of the rows' models.
void lstm_reset_rows(nam_b200_model* m, const int32_t* streams, int n, bool fresh)
{
  const size_t row = (size_t)m->state_stride;
  ensure_xfer(m, (size_t)n * row * sizeof(float));
  float* rows = reinterpret_cast<float*>(m->d_xfer);
  std::vector<StreamRef> refs((size_t)n);
  for (int i = 0; i < n; i++)
    refs[(size_t)i] = StreamRef{streams[i], m->t_base, 0, 0};
  const StreamRef* d_refs = upload_refs(m, refs, m->stream);
  if (fresh)
  {
    std::vector<int32_t> models((size_t)n);
    for (int i = 0; i < n; i++)
      models[(size_t)i] = m->stream_model[(size_t)streams[i]];
    write_lstm_initial_rows(m, rows, 0, models);
  }
  else
    copy_rows(m, rows, nullptr, m->d_state, d_refs, n, m->stream);
  if (m->opts.prewarm_on_reset)
    prewarm_blocks(m, n, n, [&](JitParams call) {
      call.state = rows;
      if (!m->is_bank)
        return launch(m, call, m->stream);
      for (int i = 0; i < n; i++)
        m->h_slots[(size_t)i] = StreamRef{i, 0u, m->stream_model[(size_t)streams[i]], call.n_frames};
      launch_with_table(m, call, n, m->stream);
    });
  copy_rows(m, m->d_state, d_refs, rows, nullptr, n, m->stream);
  mark_written(m, streams, n);
}

// ---- model banks: fresh state per model --------------------------------------------------------------------------------
// The listed streams take the fresh row of the model they are bound to (one row-copy launch whatever the mix); their
// histories then end at fresh_clock.  A bank's calls carry every stream's clock, so the streams need not be in step.
void prewarm_lstm_bank(nam_b200_model* m, bool streams);
void bank_fan_out(nam_b200_model* m, const int32_t* streams, int n, cudaStream_t st)
{
  if (m->spec.arch == Arch::LSTM && m->rows_fast_tanh != m->fast_tanh_runtime)
    prewarm_lstm_bank(m, false);
  // (an asynchronous call on another CUDA stream may still be running these streams under their previous binding: their
  // rows are rewritten after it)
  if (m->slots_used)
    CUDA_CHECK(cudaStreamWaitEvent(st, m->slots_free, 0));
  std::vector<StreamRef> refs((size_t)2 * n);
  for (int i = 0; i < n; i++)
  {
    refs[(size_t)i] = StreamRef{m->opts.max_batch + m->stream_model[(size_t)streams[i]], 0, 0, 0};
    refs[(size_t)(n + i)] = StreamRef{streams[i], 0, 0, 0};
  }
  const StreamRef* d_refs = upload_refs(m, refs, st);
  copy_rows(m, m->d_state, d_refs + n, m->d_state, d_refs, n, st);
  for (int i = 0; i < n; i++)
    m->stream_clock[(size_t)streams[i]] = m->fresh_clock;
  m->streams_identical = false;
  recount_phase(m);
}

// DSP::prewarm for a bank straight after init_state: the bank_size model rows are prewarmed together -- position k of each
// launch is model k's row, running model k -- exactly like prewarm() runs stream 0 of an ordinary handle, then every stream
// takes its model's row.
void prewarm_bank(nam_b200_model* m)
{
  const int K = m->bank_size;
  prewarm_blocks(m, K, std::max(m->opts.max_batch, K), [&](const JitParams& call) {
    for (int k = 0; k < K; k++)
      m->h_slots[(size_t)k] = StreamRef{m->opts.max_batch + k, m->t_base, k, call.n_frames};
    launch_with_table(m, call, K, m->stream);
    m->t_base += (uint32_t)call.n_frames;
  });
  m->fresh_clock = m->t_base;
  std::vector<int32_t> all((size_t)m->opts.max_batch);
  for (int s = 0; s < m->opts.max_batch; s++)
    all[(size_t)s] = s;
  bank_fan_out(m, all.data(), m->opts.max_batch, m->stream);
  CUDA_CHECK(cudaStreamSynchronize(m->stream));
}

// Why the CUDA path cannot serve this LSTM ("" when it can)
std::string lstm_refusal(const ModelSpec& s)
{
  const LstmSpec& ls = s.lstm;
  if (ls.input_size != s.in_channels) // lstm.cpp:74,111: in_channels samples land in an input_size vector
    return "LSTM input_size (" + std::to_string(ls.input_size) + ") != in_channels (" + std::to_string(s.in_channels) + ")";
  if ((int)ls.head_b.size() != s.out_channels || s.out_channels > 64)
    return "LSTM head with " + std::to_string(ls.head_b.size()) + " rows for " + std::to_string(s.out_channels) + " output channels";
  if (ls.num_layers < 1)
    return "LSTM with zero layers";
  return "";
}

// the LSTM kernels' weights: per layer W[4H][I+H] | b[4H]; then head_w | head_b
std::vector<float> lstm_blob(const ModelSpec& s)
{
  std::vector<float> blob;
  for (const auto& c : s.lstm.cells)
  {
    blob.insert(blob.end(), c.w.begin(), c.w.end());
    blob.insert(blob.end(), c.b.begin(), c.b.end());
  }
  blob.insert(blob.end(), s.lstm.head_w.begin(), s.lstm.head_w.end());
  blob.insert(blob.end(), s.lstm.head_b.begin(), s.lstm.head_b.end());
  return blob;
}

// Reset of an LSTM bank.  An LSTM keeps h, c across Reset, so each stream (streams = true) is prewarmed in place with its
// own model, as prewarm() does on an ordinary handle; in the same launches the K model rows restart from their models'
// h0 / c0 and are prewarmed: each becomes the state of a freshly created and reset handle of its model, at the current
// max_frames and prewarm_on_reset.  streams = false rebuilds the model rows alone (after a fast-tanh switch).
void prewarm_lstm_bank(nam_b200_model* m, bool streams)
{
  const int K = m->bank_size, B = m->opts.max_batch;
  std::vector<int32_t> models((size_t)K);
  for (int k = 0; k < K; k++)
    models[(size_t)k] = k;
  write_lstm_initial_rows(m, m->d_state, (size_t)B, models);
  const int n0 = streams ? B : 0, n = n0 + K;
  if (m->opts.prewarm_on_reset)
    prewarm_blocks(m, n, n, [&](const JitParams& call) {
      for (int i = 0; i < n; i++) // streams 0 .. n0 - 1, then the model rows
        m->h_slots[(size_t)i] = i < n0 ? StreamRef{i, m->stream_clock[(size_t)i], m->stream_model[(size_t)i], call.n_frames}
                                       : StreamRef{B + i - n0, m->fresh_clock, i - n0, call.n_frames};
      launch_with_table(m, call, n, m->stream);
    });
  m->rows_fast_tanh = m->fast_tanh_runtime;
  m->streams_identical = false;
  CUDA_CHECK(cudaStreamSynchronize(m->stream));
}

// Model rows k0 .. k0 + n - 1 of a bank that has been reset (nam_b200_bank_add_models, _replace_model) take the state
// nam_b200_reset would have left them in, under the current max_frames, prewarm_on_reset and fast-tanh regime; no other row,
// no clock and not t_base moves.  A WaveNet / ConvNet row starts from zeros at fresh_clock minus the prewarm's frames, so
// that it ends at fresh_clock, the clock bank_fan_out gives a stream copied from it (zero rings read the same at any
// clock, so the row equals one prewarmed at reset).  An LSTM row starts from its model's h0 / c0.  The row of an LSTM bank
// whose other rows wait for a rebuild in a new regime (rows_fast_tanh) is rebuilt with them.
void prepare_bank_rows(nam_b200_model* m, int k0, int n)
{
  const int B = m->opts.max_batch;
  const bool lstm = m->spec.arch == Arch::LSTM;
  if (lstm)
  {
    std::vector<int32_t> models((size_t)n);
    for (int i = 0; i < n; i++)
      models[(size_t)i] = k0 + i;
    write_lstm_initial_rows(m, m->d_state, (size_t)(B + k0), models);
  }
  else
    CUDA_CHECK(cudaMemsetAsync(m->d_state + (size_t)(B + k0) * m->state_stride, 0, (size_t)n * m->state_stride * sizeof(float),
                               m->stream));
  if (m->opts.prewarm_on_reset)
  {
    const int bs = std::max(m->max_frames, 1), ps = m->spec.prewarm_samples;
    const uint32_t frames = ps > 0 ? (uint32_t)((ps + bs - 1) / bs) * (uint32_t)bs : 0u;
    uint32_t clock = lstm ? m->fresh_clock : m->fresh_clock - frames;
    prewarm_blocks(m, n, n, [&](const JitParams& call) {
      for (int i = 0; i < n; i++)
        m->h_slots[(size_t)i] = StreamRef{B + k0 + i, clock, k0 + i, call.n_frames};
      launch_with_table(m, call, n, m->stream);
      clock += lstm ? 0u : (uint32_t)call.n_frames;
    });
  }
  CUDA_CHECK(cudaStreamSynchronize(m->stream));
}

// ---- which kernel serves a model ---------------------------------------------------------------------------------------
enum class KernelFamily
{
  Fused, // WaveNet on the fused kernel
  General, // WaveNet on the general kernel
  ConvNet,
  Lstm,
  Linear
};

// The kernel a handle of a (non-container) model runs, and what the host prepares for it; or, when code != NAM_B200_OK,
// create's refusal.  A refusal keeps the plans it made.
struct KernelChoice
{
  int code = NAM_B200_OK;
  std::string refusal;
  KernelFamily family = KernelFamily::Fused;
  WaveNetPlan plan; // WaveNet (the fused kernel's; for the general family, plan.why_not says why the fused kernel declined)
  GenericPlan gplan; // general WaveNet, ConvNet
  std::vector<float> blob;
  long state_stride = 0;
  double flops_per_frame = 0.0;
  int variant = 0;
};

// kernel_geometry (nam_b200_options): 0 default, 1 = FFMA 128-thread, 2 = FFMA 256-thread, 3 = tensor-core (none on sm_90a),
// 4 = the general kernel
KernelChoice choose_kernel(const ModelSpec& s, int kernel_geometry)
{
  KernelChoice c;
  auto refuse = [&](std::string why) {
    c.code = NAM_B200_ERR_UNSUPPORTED;
    c.refusal = std::move(why);
    return c;
  };
  switch (s.arch)
  {
    case Arch::WaveNet:
    {
      WaveNetPlan& p = c.plan;
      p = plan_wavenet(s);
      if (p.eligible && !(s.in_channels == 1 && s.out_channels == 1))
      {
        p.eligible = false;
        p.why_not = "multi-channel in / out";
      }
      if (p.eligible && kernel_geometry != 3 && wavenet_smem_bytes(p, kernel_geometry == 1 ? 0 : 1) > 227 * 1024)
      {
        // e.g. > ~50 layers of 16 channels: the general kernel keeps such weights in global memory
        p.eligible = false;
        p.why_not = "packed weights + tile exceed the 227 KB of shared memory of the fused kernel";
      }
      if (!p.eligible || kernel_geometry == 4)
      {
        // outside the fused families (or asked for explicitly): the general kernel
        c.gplan = plan_generic(s);
        if (!c.gplan.eligible)
          return refuse("WaveNet not supported on the CUDA path: fused kernel: "
                        + (p.eligible ? std::string("(eligible)") : p.why_not) + "; general kernel: " + c.gplan.why_not);
        c.family = KernelFamily::General;
        c.blob = c.gplan.weights;
        c.state_stride = c.gplan.state_floats;
        c.flops_per_frame = 2.0 * c.gplan.macs_per_frame;
        c.variant = 9000;
        return c;
      }
      if (kernel_geometry == 3)
        return refuse("tensor-core WaveNet kernel: this sm_90a library has none (use kernel_geometry 0, 1, 2 or 4)");
      c.family = KernelFamily::Fused;
      c.blob = p.blob;
      c.state_stride = p.state_floats;
      c.flops_per_frame = 2.0 * p.macs_per_frame;
      c.variant = p.cp[0] * 100 + (p.n_arrays > 1 ? p.cp[1] : 0);
      return c;
    }
    case Arch::LSTM:
    {
      const LstmSpec& ls = s.lstm;
      const std::string why = lstm_refusal(s);
      if (!why.empty())
        return refuse(why);
      double macs = 0.0;
      for (const auto& cell : ls.cells)
        macs += 4.0 * cell.hidden * (cell.input_size + cell.hidden);
      macs += (double)ls.hidden * s.out_channels;
      c.family = KernelFamily::Lstm;
      c.blob = lstm_blob(s);
      c.state_stride = ((long)ls.num_layers * 2 * ls.hidden + 3) & ~3L;
      c.flops_per_frame = 2.0 * macs;
      c.variant = 2000 + ls.hidden;
      return c;
    }
    case Arch::Linear:
      if (!(s.in_channels == 1 && s.out_channels == 1))
        return refuse("Linear on the CUDA path is mono in / mono out (model has " + std::to_string(s.in_channels) + " in, "
                      + std::to_string(s.out_channels) + " out channels)");
      c.family = KernelFamily::Linear;
      c.blob = s.linear.impulse;
      c.state_stride = ((long)std::max(s.linear.receptive_field - 1, 1) + 3) & ~3L;
      c.flops_per_frame = 2.0 * s.linear.receptive_field;
      c.variant = 3000;
      return c;
    case Arch::ConvNet:
      c.gplan = plan_convnet(s);
      if (!c.gplan.eligible)
        return refuse("ConvNet not supported on the CUDA path: " + c.gplan.why_not);
      c.family = KernelFamily::ConvNet;
      c.blob = c.gplan.weights;
      c.state_stride = std::max(c.gplan.state_floats, 4L);
      c.flops_per_frame = 2.0 * c.gplan.macs_per_frame;
      c.variant = 9500;
      return c;
    default: return refuse("no CUDA kernel for architecture " + s.architecture);
  }
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

    KernelChoice c = choose_kernel(m->spec, m->opts.kernel_geometry);
    if (c.code != NAM_B200_OK)
      return fail(c.code, c.refusal);
    m->plan = std::move(c.plan);
    m->gplan = std::move(c.gplan);
    m->use_generic = c.family == KernelFamily::General;
    m->state_stride = c.state_stride;
    m->flops_per_frame = c.flops_per_frame;
    m->variant = c.variant;
    switch (c.family)
    {
      case KernelFamily::General:
        setup_generic_spec_kernel(m.get()); // throws when jit = 1 and the specialised general kernel cannot be had
        CUDA_CHECK(cudaMalloc(&m->d_glayers, std::max<size_t>(m->gplan.layers.size(), 1) * sizeof(GLayer)));
        CUDA_CHECK(cudaMemcpy(m->d_glayers, m->gplan.layers.data(), m->gplan.layers.size() * sizeof(GLayer),
                              cudaMemcpyHostToDevice));
        break;
      case KernelFamily::Fused:
        m->wn_geometry = (m->opts.kernel_geometry == 1) ? 0 : 1;
        setup_spec_kernel(m.get());
        break;
      case KernelFamily::Lstm: setup_lstm_spec_kernel(m.get()); break;
      default: break;
    }
    std::vector<float> blob = std::move(c.blob);
    m->n_weight_floats = blob.size();
    const size_t alloc_floats = (blob.size() + 3) & ~(size_t)3;
    blob.resize(alloc_floats, 0.0f);
    CUDA_CHECK(cudaMalloc(&m->d_weights, alloc_floats * sizeof(float)));
    CUDA_CHECK(cudaMemcpy(m->d_weights, blob.data(), alloc_floats * sizeof(float), cudaMemcpyHostToDevice));
    const size_t state_total = (size_t)m->state_stride * m->opts.max_batch;
    CUDA_CHECK(cudaMalloc(&m->d_state, std::max<size_t>(state_total, 4) * sizeof(float)));
    if (m->spec.arch == Arch::Linear)
      CUDA_CHECK(cudaMalloc(&m->d_state_tmp, std::max<size_t>(state_total, 4) * sizeof(float)));
    m->stream_clock.assign((size_t)m->opts.max_batch, 0u);
    m->stream_flips.assign((size_t)m->opts.max_batch, 0u);
    m->stream_model.assign((size_t)m->opts.max_batch, 0);
    m->h_slots.assign((size_t)m->opts.max_batch, StreamRef{0, 0u, 0, 0});
    CUDA_CHECK(cudaMalloc(&m->d_slots, (size_t)m->opts.max_batch * sizeof(StreamRef)));
    CUDA_CHECK(cudaEventCreateWithFlags(&m->slots_free, cudaEventDisableTiming));
    try
    {
      setup_state_records(m.get());
    }
    catch (const CudaError&)
    {
      throw;
    }
    catch (const std::exception& ex)
    {
      m->state_error = ex.what();
    }
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
  if (n_frames < 0 || n_frames > call_max_frames(m))
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "n_frames " + std::to_string(n_frames) + " exceeds max_frames "
                                                 + std::to_string(call_max_frames(m)) + " of the last reset");
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
    float* hout = m->h_pin + (size_t)staging_frames(m) * std::max(ci, co);
    for (size_t c = 0; c < ci; c++)
      for (size_t i = 0; i < n; i++)
        hin[c * n + i] = (float)input[c][i];
    if ((ci + co) * n <= kZeroCopyFloats && m->h_pin_dev != nullptr)
    {
      float* din = m->h_pin_dev;
      float* dout = m->h_pin_dev + (hout - hin);
      m->flag_pending = false;
      // (a converting handle's last launch is the history update, not the model's: no doorbell)
      const bool doorbell = m->h_flag_dev != nullptr && n_frames <= 128 && !m->opts_timing_events && !m->rs.active;
      if (!doorbell)
        CUDA_CHECK(cudaEventRecord(m->ev0, m->stream));
      run_call(m, din, dout, 1, n_frames, (long)(ci * n), (long)(co * n), m->stream);
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
      run_call(m, m->d_in, m->d_out, 1, n_frames, (long)(ci * n), (long)(co * n), m->stream);
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

// ---- argument checks of the stream-state calls: all on the host, before anything is launched ---------------------------
int check_state_calls(nam_b200_model* m, const char* fn)
{
  if (!m->state_error.empty())
    return fail(NAM_B200_ERR_UNSUPPORTED, std::string(fn) + ": no per-stream state records for this handle: " + m->state_error);
  if (!m->is_reset)
    return fail(NAM_B200_ERR_STATE, std::string(fn) + " called before reset");
  return NAM_B200_OK;
}

int check_stream_list(const nam_b200_model* m, const int32_t* idx, int n, const char* what, bool distinct)
{
  if (n < 0)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, std::string(what) + ": negative stream count " + std::to_string(n));
  if (n > 0 && !idx)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, std::string(what) + ": null stream list");
  std::vector<char> seen(distinct ? (size_t)m->opts.max_batch : 0, 0);
  // (the message is only built for the failing entry: a per-call table of thousands of streams passes through here)
  auto at = [&](int i) { return std::string(what) + "[" + std::to_string(i) + "] = " + std::to_string(idx[i]); };
  for (int i = 0; i < n; i++)
  {
    const int32_t s = idx[i];
    if (s < 0 || s >= m->opts.max_batch)
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, at(i) + ": stream index outside [0, max_batch=" + std::to_string(m->opts.max_batch) + ")");
    if (distinct && seen[(size_t)s]++)
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, at(i) + ": duplicate destination stream");
  }
  return NAM_B200_OK;
}

// a record's header word 3 must hold the handle's conversion ratio (0 when it converts nothing)
int check_record_ratio(const nam_b200_model* m, const StateRecordHeader& h, const std::string& at)
{
  if (h.reserved == rs_ratio(m))
    return NAM_B200_OK;
  auto ratio = [](uint32_t r) { return r ? std::to_string(r >> 16) + "/" + std::to_string(r & 0xffffu) : std::string("none"); };
  return fail(NAM_B200_ERR_INVALID_ARGUMENT, at + "resample ratio (header word 3) " + ratio(h.reserved) + ", this handle's is "
                                               + ratio(rs_ratio(m)) + " (model / host rate, as of its last reset)");
}

// `incoming`: records to import -- a stride too small for this handle's record is first checked for a conversion ratio
// that differs from the handle's (a record of another rate pair has another size), so that the refusal names the cause
int check_records(const nam_b200_model* m, const void* buf, int n, int64_t stride, bool device, bool incoming = false)
{
  if (n > 0 && !buf)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null record buffer");
  const size_t rb = record_bytes(m);
  if (stride < (int64_t)rb && incoming && n > 0 && stride >= kStateHeaderBytes)
  {
    StateRecordHeader h;
    if (device)
      CUDA_CHECK(cudaMemcpy(&h, buf, sizeof h, cudaMemcpyDeviceToHost));
    else
      std::memcpy(&h, buf, sizeof h);
    if (std::memcmp(h.magic, "NAMS", 4) == 0 && check_record_ratio(m, h, "record 0: ") != NAM_B200_OK)
      return NAM_B200_ERR_INVALID_ARGUMENT;
  }
  if (stride < (int64_t)rb)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "record_stride " + std::to_string(stride) + " is smaller than the record ("
                                                 + std::to_string(rb) + " bytes)");
  if (device && (stride % 4 != 0 || reinterpret_cast<uintptr_t>(buf) % 4 != 0))
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "device records must be 4-byte aligned (record_stride " + std::to_string(stride) + ")");
  return NAM_B200_OK;
}

// the header of record i (for stream `stream`) must be this model's -- a bank's: one of its models', *model receives the
// lowest such index (0 on an ordinary handle)
int check_record_header(const nam_b200_model* m, const unsigned char* rec, int i, int stream, int* model = nullptr)
{
  if (model)
    *model = 0;
  StateRecordHeader h;
  std::memcpy(&h, rec, sizeof h);
  const StateRecordHeader& want = m->record_header;
  const std::string at = "record " + std::to_string(i) + " (stream " + std::to_string(stream) + "): ";
  char hex[2][24];
  std::snprintf(hex[0], sizeof hex[0], "%016llx", (unsigned long long)h.fingerprint);
  std::snprintf(hex[1], sizeof hex[1], "%016llx", (unsigned long long)want.fingerprint);
  if (std::memcmp(h.magic, "NAMS", 4) != 0)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, at + "magic is not \"NAMS\": not a stream state record");
  if (h.version != kStateRecordVersion)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, at + "format version " + std::to_string(h.version) + " (this library reads "
                                                 + std::to_string(kStateRecordVersion) + ")");
  if (h.architecture != want.architecture)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, at + "architecture " + std::to_string(h.architecture) + ", the model's is "
                                                 + std::to_string(want.architecture));
  if (check_record_ratio(m, h, at) != NAM_B200_OK)
    return NAM_B200_ERR_INVALID_ARGUMENT;
  const uint64_t payload = want.payload_floats + (uint64_t)rs_record_floats(m);
  if (h.payload_floats != payload)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, at + "payload float count " + std::to_string(h.payload_floats)
                                                 + ", the model's record holds " + std::to_string(payload));
  if (m->is_bank)
  {
    for (int k = 0; k < m->bank_size; k++)
      if (h.fingerprint == m->bank_headers[(size_t)k].fingerprint)
      {
        if (model)
          *model = k;
        return NAM_B200_OK;
      }
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, at + "model fingerprint " + hex[0] + " is none of the "
                                                 + std::to_string(m->bank_size) + " models of this bank");
  }
  if (h.fingerprint != want.fingerprint)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, at + "model fingerprint " + hex[0] + " is not this model's (" + hex[1]
                                                 + "): a record of another model, or of another slimmable size");
  return NAM_B200_OK;
}

// The host-buffer entries (nam_b200_process_f32, nam_b200_process_streams_f32): `streams` (n entries) or, when nullptr,
// streams [0, n).  Large WaveNet batches are pipelined in chunks of whole kernel waves so that the copies of chunk c+1 /
// c-1 overlap the kernel of chunk c (the kernel is compute-bound; the copies would otherwise add ~18 %); a chunk of a table
// call is a sub-range of the table.  Returns once `out` is filled.
// `counts` (nam_b200_process_streams_ragged_f32, with `streams`): row i runs counts[i] <= n_frames frames, n_frames stays
// the staging pitch.  The kernels never write past a row's count, so when some row is short the output staging is zeroed
// first and the padding arrives as zeros.
void process_host(nam_b200_model* m, const int32_t* streams, int n, const float* in, float* out, int n_frames, int64_t in_stride,
                  int64_t out_stride, const int32_t* counts = nullptr)
{
  const size_t ci = (size_t)m->spec.in_channels, co = (size_t)m->spec.out_channels;
  const size_t row = (size_t)n_frames * sizeof(float);
  const bool padded = counts != nullptr && std::any_of(counts, counts + n, [&](int32_t c) { return c < n_frames; });
  const int chunk = wavenet_chunk_streams(m);
  if (chunk > 0 && n >= 2 * chunk && (size_t)n * row >= ((size_t)8 << 20) && !m->rs.active)
  {
    const int n_chunks = (n + chunk - 1) / chunk;
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
    const bool table = streams != nullptr || prefix_needs_table(m, n);
    CUDA_CHECK(cudaEventRecord(m->ev0, m->stream));
    const StreamRef* slots = table ? upload_slots(m, streams, n, n_frames, counts, m->stream) : nullptr;
    for (int c = 0; c < n_chunks; c++)
    {
      const int s0 = c * chunk, nb = std::min(chunk, n - s0);
      float* din = m->d_in + (size_t)s0 * n_frames;
      float* dout = m->d_out + (size_t)s0 * n_frames;
      cudaEvent_t e_in = m->chunk_events[2 * c], e_k = m->chunk_events[2 * c + 1];
      CUDA_CHECK(cudaMemcpy2DAsync(din, row, in + (size_t)s0 * in_stride, (size_t)in_stride * sizeof(float), row,
                                   (size_t)nb, cudaMemcpyHostToDevice, m->copy_in));
      CUDA_CHECK(cudaEventRecord(e_in, m->copy_in));
      CUDA_CHECK(cudaStreamWaitEvent(m->stream, e_in, 0));
      if (padded)
        CUDA_CHECK(cudaMemsetAsync(dout, 0, (size_t)nb * row, m->stream));
      // (without a table, the chunk's positions are state rows s0 ..)
      float* const state = slots ? m->d_state : m->d_state + (size_t)s0 * (size_t)m->state_stride;
      launch(m, jit_params(m, state, din, dout, n_frames, n_frames, nb, n_frames, slots ? slots + s0 : nullptr), m->stream);
      CUDA_CHECK(cudaEventRecord(e_k, m->stream));
      CUDA_CHECK(cudaStreamWaitEvent(m->copy_out, e_k, 0));
      CUDA_CHECK(cudaMemcpy2DAsync(out + (size_t)s0 * out_stride, (size_t)out_stride * sizeof(float), dout, row, row,
                                   (size_t)nb, cudaMemcpyDeviceToHost, m->copy_out));
    }
    if (table)
      finish_table_call(m, n, n_frames, m->stream);
    else
      finish_contiguous_call(m, n, n_frames);
    CUDA_CHECK(cudaEventRecord(m->ev1, m->stream));
    CUDA_CHECK(cudaStreamSynchronize(m->copy_out));
    CUDA_CHECK(cudaStreamSynchronize(m->stream));
    m->timing_valid = true;
    return;
  }
  // (multi-channel models: a stream's row is its channel planes back to back)
  CUDA_CHECK(cudaMemcpy2DAsync(m->d_in, ci * row, in, (size_t)in_stride * sizeof(float), ci * row, (size_t)n,
                               cudaMemcpyHostToDevice, m->stream));
  if (padded)
    CUDA_CHECK(cudaMemsetAsync(m->d_out, 0, (size_t)n * co * row, m->stream));
  CUDA_CHECK(cudaEventRecord(m->ev0, m->stream));
  run_call(m, m->d_in, m->d_out, n, n_frames, (long)(ci * n_frames), (long)(co * n_frames), m->stream, streams, counts);
  CUDA_CHECK(cudaEventRecord(m->ev1, m->stream));
  CUDA_CHECK(cudaMemcpy2DAsync(out, (size_t)out_stride * sizeof(float), m->d_out, co * row, co * row, (size_t)n,
                               cudaMemcpyDeviceToHost, m->stream));
  CUDA_CHECK(cudaStreamSynchronize(m->stream));
  m->timing_valid = true;
}

// nam_b200_process_streams_f32(_device): everything checked on the host before anything is queued
int check_process_streams_args(const nam_b200_model* m, const char* fn, const int32_t* streams, int n, const void* in,
                               const void* out, int n_frames, int64_t in_stride, int64_t out_stride)
{
  const std::string f(fn);
  if (!m->is_reset)
    return fail(NAM_B200_ERR_STATE, f + " called before reset");
  if (n < 0 || n > m->opts.max_batch)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT,
                f + ": n = " + std::to_string(n) + " outside [0, max_batch=" + std::to_string(m->opts.max_batch) + "]");
  if (n_frames < 0 || n_frames > call_max_frames(m))
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, f + ": n_frames " + std::to_string(n_frames) + " outside [0, max_frames="
                                                 + std::to_string(call_max_frames(m)) + "] of the last reset");
  if (n == 0 || n_frames == 0)
    return NAM_B200_OK;
  if (!in || !out)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, f + ": null audio buffer");
  const int rc = check_stream_list(m, streams, n, (f + ": streams").c_str(), true);
  if (rc != NAM_B200_OK)
    return rc;
  const int64_t ci = m->spec.in_channels, co = m->spec.out_channels;
  if (in_stride < ci * n_frames)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, f + ": in_stride " + std::to_string(in_stride) + " < in_channels x n_frames = "
                                                 + std::to_string(ci * n_frames));
  if (out_stride < co * n_frames)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, f + ": out_stride " + std::to_string(out_stride)
                                                 + " < out_channels x n_frames = " + std::to_string(co * n_frames));
  return NAM_B200_OK;
}

// nam_b200_process_streams_ragged_f32(_device): the per-row counts, then the checks of a process_streams call of
// *n_max = max(n_frames[i]) frames
int check_ragged_args(const nam_b200_model* m, const char* fn, const int32_t* streams, int n, const int32_t* n_frames,
                      const void* in, const void* out, int64_t in_stride, int64_t out_stride, int* n_max)
{
  const std::string f(fn);
  *n_max = 0;
  if (!m->is_reset)
    return fail(NAM_B200_ERR_STATE, f + " called before reset");
  if (n > 0 && n <= m->opts.max_batch)
  {
    if (!n_frames)
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, f + ": null n_frames");
    for (int i = 0; i < n; i++)
    {
      if (n_frames[i] < 0 || n_frames[i] > call_max_frames(m))
        return fail(NAM_B200_ERR_INVALID_ARGUMENT, f + ": n_frames[" + std::to_string(i) + "] = " + std::to_string(n_frames[i])
                                                     + " outside [0, max_frames=" + std::to_string(call_max_frames(m))
                                                     + "] of the last reset");
      *n_max = std::max(*n_max, (int)n_frames[i]);
    }
  }
  return check_process_streams_args(m, fn, streams, n, in, out, *n_max, in_stride, out_stride);
}

// host records go through device staging in groups of at most this many bytes
constexpr size_t kRecordStagingBytes = (size_t)64 << 20;

// ---- model banks: which documents can share one handle ---------------------------------------------------------------
// Model 0 chooses the family: WaveNets served by the fused kernel, WaveNets served by the general kernel, ConvNets, or
// LSTMs.  Models 1.. must be of model 0's architecture and family and match it in everything but their weights (a
// WaveNet's head_scale, the last weight, and an LSTM's h0 / c0 and head included): the same expected sample rate (as
// ContainerModel requires of its sub-models), the same config object, and the same packed form apart from the blob's values
// (WaveNetPlan, GenericPlan) or, for an LSTM, the same channels, layers and sizes.
struct BankCheck
{
  int code = NAM_B200_OK;
  std::string reason; // names the first offending model and the field
  KernelFamily family = KernelFamily::Fused;
  std::vector<WaveNetPlan> plans; // fused family
  std::vector<GenericPlan> gplans; // general WaveNets and ConvNets
};

// "" when model k (spec s, plan p) matches model 0 (s0, p0), else the first difference
std::string bank_difference(int k, const ModelSpec& s, const WaveNetPlan& p, const ModelSpec& s0, const WaveNetPlan& p0)
{
  const std::string mk = "model " + std::to_string(k) + " differs from model 0 in ";
  auto num = [](double v) { return json::number_to_string(v); };
  auto differ = [&](const std::string& field, double a, double b) { return mk + field + " (" + num(a) + " vs " + num(b) + ")"; };
  if (!(s.sample_rate == s0.sample_rate))
    return differ("expected sample_rate", s.sample_rate, s0.sample_rate);
  const WaveNetSpec &w = s.wavenet, &w0 = s0.wavenet;
  if (w.arrays.size() != w0.arrays.size())
    return differ("the number of layer arrays", (double)w.arrays.size(), (double)w0.arrays.size());
  for (size_t a = 0; a < w.arrays.size(); a++)
  {
    const ArraySpec &A = w.arrays[a], &A0 = w0.arrays[a];
    const std::string at = "array " + std::to_string(a) + " ";
    const struct
    {
      const char* name;
      int v, v0;
    } fields[] = {{"input_size", A.input_size, A0.input_size},
                  {"condition_size", A.condition_size, A0.condition_size},
                  {"channels", A.channels, A0.channels},
                  {"bottleneck", A.bottleneck, A0.bottleneck},
                  {"head_size", A.head_size, A0.head_size},
                  {"head kernel_size", A.head_kernel, A0.head_kernel},
                  {"head dilation", A.head_dilation, A0.head_dilation},
                  {"head_bias", A.head_bias ? 1 : 0, A0.head_bias ? 1 : 0},
                  {"number of layers (dilations)", (int)A.layers.size(), (int)A0.layers.size()}};
    for (const auto& f : fields)
      if (f.v != f.v0)
        return differ(at + f.name, f.v, f.v0);
    for (size_t l = 0; l < A.layers.size(); l++)
    {
      const LayerSpec &L = A.layers[l], &L0 = A0.layers[l];
      const std::string lt = at + "layer " + std::to_string(l) + " ";
      if (L.conv.kernel != L0.conv.kernel)
        return differ(lt + "kernel_size", L.conv.kernel, L0.conv.kernel);
      if (L.conv.dilation != L0.conv.dilation)
        return differ(lt + "dilation", L.conv.dilation, L0.conv.dilation);
      if (L.gating != L0.gating)
        return differ(lt + "gating", (int)L.gating, (int)L0.gating);
      if (L.act.type != L0.act.type)
        return differ(lt + "activation", (int)L.act.type, (int)L0.act.type);
      if (L.act.slope != L0.act.slope || L.act.slopes != L0.act.slopes || L.act.min_val != L0.act.min_val
          || L.act.max_val != L0.act.max_val || L.act.min_slope != L0.act.min_slope || L.act.max_slope != L0.act.max_slope)
        return mk + lt + "activation parameters";
    }
  }
  // the packed form (padded channels, ring layout, descriptors, blob length) -- equal whenever the above is, kept as the
  // statement of what the kernels rely on
  bool same = p.n_arrays == p0.n_arrays && p.blob.size() == p0.blob.size() && p.state_floats == p0.state_floats
              && std::equal(p.cp, p.cp + kMaxArrays, p0.cp) && std::equal(p.creal, p.creal + kMaxArrays, p0.creal)
              && p.arrays.size() == p0.arrays.size() && p.layers.size() == p0.layers.size();
  same = same && std::memcmp(p.arrays.data(), p0.arrays.data(), p.arrays.size() * sizeof(ArrayDesc)) == 0
         && std::memcmp(p.layers.data(), p0.layers.data(), p.layers.size() * sizeof(LayerDesc)) == 0;
  if (!same)
    return mk + "the packed kernel layout (descriptors, rings or blob length)";
  if (s.config_fingerprint != s0.config_fingerprint)
    return mk + "its config object (apart from the weights and head_scale)";
  return "";
}

// "" when LSTM k (spec s) matches model 0 (s0), else the first difference
std::string lstm_bank_difference(int k, const ModelSpec& s, const ModelSpec& s0)
{
  const std::string mk = "model " + std::to_string(k) + " differs from model 0 in ";
  auto differ = [&](const std::string& field, double a, double b) {
    return mk + field + " (" + json::number_to_string(a) + " vs " + json::number_to_string(b) + ")";
  };
  if (!(s.sample_rate == s0.sample_rate))
    return differ("expected sample_rate", s.sample_rate, s0.sample_rate);
  const struct
  {
    const char* name;
    int v, v0;
  } fields[] = {{"prewarm samples", s.prewarm_samples, s0.prewarm_samples},
                {"in_channels", s.in_channels, s0.in_channels},
                {"out_channels", s.out_channels, s0.out_channels},
                {"num_layers", s.lstm.num_layers, s0.lstm.num_layers},
                {"input_size", s.lstm.input_size, s0.lstm.input_size},
                {"hidden_size", s.lstm.hidden, s0.lstm.hidden}};
  for (const auto& f : fields)
    if (f.v != f.v0)
      return differ(f.name, f.v, f.v0);
  if (s.config_fingerprint != s0.config_fingerprint)
    return mk + "its config object (apart from the weights)";
  return "";
}

// "" when the WaveNet w (model k's, or its condition_dsp's) has the shape of w0, else the first difference -- the fields the
// general kernel's descriptors are made of, named as the config names them; `at` prefixes the field ("condition_dsp ")
std::string general_wavenet_difference(const std::string& mk, const std::string& at, const WaveNetSpec& w, const WaveNetSpec& w0)
{
  auto differ = [&](const std::string& field, double a, double b) {
    return mk + at + field + " (" + json::number_to_string(a) + " vs " + json::number_to_string(b) + ")";
  };
  if (w.in_channels != w0.in_channels)
    return differ("in_channels", w.in_channels, w0.in_channels);
  if (w.arrays.size() != w0.arrays.size())
    return differ("the number of layer arrays", (double)w.arrays.size(), (double)w0.arrays.size());
  auto act_difference = [&](const std::string& where, const ActSpec& a, const ActSpec& a0) -> std::string {
    if (a.type != a0.type)
      return differ(where, (int)a.type, (int)a0.type);
    if (a.slopes.size() != a0.slopes.size())
      return differ(where + " PReLU slope count", (double)a.slopes.size(), (double)a0.slopes.size());
    if (a.slope != a0.slope || a.min_val != a0.min_val || a.max_val != a0.max_val || a.min_slope != a0.min_slope
        || a.max_slope != a0.max_slope)
      return mk + at + where + " parameters";
    return "";
  };
  for (size_t a = 0; a < w.arrays.size(); a++)
  {
    const ArraySpec &A = w.arrays[a], &A0 = w0.arrays[a];
    const std::string ar = "array " + std::to_string(a) + " ";
    const struct
    {
      const char* name;
      int v, v0;
    } fields[] = {{"input_size", A.input_size, A0.input_size},
                  {"condition_size", A.condition_size, A0.condition_size},
                  {"channels", A.channels, A0.channels},
                  {"bottleneck", A.bottleneck, A0.bottleneck},
                  {"head_size", A.head_size, A0.head_size},
                  {"head kernel_size", A.head_kernel, A0.head_kernel},
                  {"head dilation", A.head_dilation, A0.head_dilation},
                  {"head_bias", A.head_bias ? 1 : 0, A0.head_bias ? 1 : 0},
                  {"groups_input", A.groups_input, A0.groups_input},
                  {"groups_input_mixin", A.groups_input_mixin, A0.groups_input_mixin},
                  {"layer1x1 active", A.l1x1_active ? 1 : 0, A0.l1x1_active ? 1 : 0},
                  {"layer1x1 groups", A.l1x1_groups, A0.l1x1_groups},
                  {"head1x1 active", A.h1x1_active ? 1 : 0, A0.h1x1_active ? 1 : 0},
                  {"head1x1 out_channels", A.h1x1_out, A0.h1x1_out},
                  {"head1x1 groups", A.h1x1_groups, A0.h1x1_groups},
                  {"number of layers (dilations)", (int)A.layers.size(), (int)A0.layers.size()}};
    for (const auto& f : fields)
      if (f.v != f.v0)
        return differ(ar + f.name, f.v, f.v0);
    for (size_t l = 0; l < A.layers.size(); l++)
    {
      const LayerSpec &L = A.layers[l], &L0 = A0.layers[l];
      const std::string lt = ar + "layer " + std::to_string(l) + " ";
      if (L.conv.kernel != L0.conv.kernel)
        return differ(lt + "kernel_size", L.conv.kernel, L0.conv.kernel);
      if (L.conv.dilation != L0.conv.dilation)
        return differ(lt + "dilation", L.conv.dilation, L0.conv.dilation);
      if (L.conv.groups != L0.conv.groups)
        return differ(lt + "groups", L.conv.groups, L0.conv.groups);
      if (L.gating != L0.gating)
        return differ(lt + "gating mode", (int)L.gating, (int)L0.gating);
      std::string d = act_difference(lt + "activation", L.act, L0.act);
      if (d.empty() && L.gating != Gating::None)
        d = act_difference(lt + "secondary activation", L.sec_act, L0.sec_act);
      if (!d.empty())
        return d;
      for (int f = 0; f < F_COUNT; f++)
      {
        const FilmSpec &F = L.film[f], &F0 = L0.film[f];
        const std::string ft = lt + "FiLM site " + std::to_string(f) + " ";
        if (F.active != F0.active)
          return differ(ft + "active", F.active ? 1 : 0, F0.active ? 1 : 0);
        if (F.shift != F0.shift)
          return differ(ft + "shift", F.shift ? 1 : 0, F0.shift ? 1 : 0);
        if (F.groups != F0.groups)
          return differ(ft + "groups", F.groups, F0.groups);
      }
    }
  }
  if (w.with_head != w0.with_head)
    return differ("post-stack head", w.with_head ? 1 : 0, w0.with_head ? 1 : 0);
  if (w.with_head)
  {
    const PostHeadSpec &H = w.post_head, &H0 = w0.post_head;
    if (H.convs.size() != H0.convs.size() || H.channels != H0.channels || H.out_channels != H0.out_channels)
      return mk + at + "the post-stack head's convolutions";
    for (size_t i = 0; i < H.convs.size(); i++)
      if (H.convs[i].kernel != H0.convs[i].kernel || H.convs[i].dilation != H0.convs[i].dilation)
        return mk + at + "the post-stack head's convolutions";
    const std::string d = act_difference("post-stack head activation", H.act, H0.act);
    if (!d.empty())
      return d;
  }
  if ((w.condition_dsp != nullptr) != (w0.condition_dsp != nullptr))
    return differ("condition_dsp", w.condition_dsp ? 1 : 0, w0.condition_dsp ? 1 : 0);
  if (w.condition_dsp)
  {
    const ModelSpec &c = *w.condition_dsp, &c0 = *w0.condition_dsp;
    if (c.out_channels != c0.out_channels)
      return differ("condition_dsp out_channels", c.out_channels, c0.out_channels);
    return general_wavenet_difference(mk, at + "condition_dsp ", c.wavenet, c0.wavenet);
  }
  return "";
}

// "" when general WaveNet or ConvNet k (spec s, plan p) matches model 0 (s0, p0), else the first difference
std::string general_bank_difference(int k, const ModelSpec& s, const GenericPlan& p, const ModelSpec& s0, const GenericPlan& p0)
{
  const std::string mk = "model " + std::to_string(k) + " differs from model 0 in ";
  auto differ = [&](const std::string& field, double a, double b) {
    return mk + field + " (" + json::number_to_string(a) + " vs " + json::number_to_string(b) + ")";
  };
  if (!(s.sample_rate == s0.sample_rate))
    return differ("expected sample_rate", s.sample_rate, s0.sample_rate);
  const struct
  {
    const char* name;
    int v, v0;
  } fields[] = {{"in_channels", s.in_channels, s0.in_channels}, {"out_channels", s.out_channels, s0.out_channels}};
  for (const auto& f : fields)
    if (f.v != f.v0)
      return differ(f.name, f.v, f.v0);
  bool same = p.weights.size() == p0.weights.size() && p.state_floats == p0.state_floats;
  if (s.arch == Arch::ConvNet)
  {
    const ConvNetSpec &c = s.convnet, &c0 = s0.convnet;
    if (c.channels != c0.channels)
      return differ("channels", c.channels, c0.channels);
    if (c.blocks.size() != c0.blocks.size())
      return differ("the number of blocks (dilations)", (double)c.blocks.size(), (double)c0.blocks.size());
    for (size_t b = 0; b < c.blocks.size(); b++)
      if (c.blocks[b].conv.dilation != c0.blocks[b].conv.dilation)
        return differ("block " + std::to_string(b) + " dilation", c.blocks[b].conv.dilation, c0.blocks[b].conv.dilation);
    if (c.batchnorm != c0.batchnorm)
      return differ("batchnorm", c.batchnorm ? 1 : 0, c0.batchnorm ? 1 : 0);
    if (c.groups != c0.groups)
      return differ("groups", c.groups, c0.groups);
    if (c.act.type != c0.act.type)
      return differ("activation", (int)c.act.type, (int)c0.act.type);
    // (GConvNet is plain 4-byte fields: no padding to compare)
    same = same && std::memcmp(&p.convnet, &p0.convnet, sizeof(GConvNet)) == 0;
  }
  else
  {
    const std::string d = general_wavenet_difference(mk, "", s.wavenet, s0.wavenet);
    if (!d.empty())
      return d;
    // the packed form apart from the weights and the two output scales (which a bank's kernel reads from each blob)
    GNet n = p.net, n0 = p0.net, c = p.cond, c0 = p0.cond;
    n.head_scale = n0.head_scale = c.head_scale = c0.head_scale = 0.0f;
    same = same && p.has_cond == p0.has_cond && std::memcmp(&n, &n0, sizeof(GNet)) == 0
           && std::memcmp(&c, &c0, sizeof(GNet)) == 0 && p.layers.size() == p0.layers.size()
           && std::memcmp(p.layers.data(), p0.layers.data(), p.layers.size() * sizeof(GLayer)) == 0;
  }
  // (after the fields above: the receptive field decides it)
  if (s.prewarm_samples != s0.prewarm_samples)
    return differ("prewarm samples", s.prewarm_samples, s0.prewarm_samples);
  if (!same)
    return mk + "the packed kernel layout (descriptors, rings or blob length)";
  if (s.config_fingerprint != s0.config_fingerprint)
    return mk + "its config object (apart from the weights and head_scale)";
  return "";
}

// specs[0] is model 0; specs[k] (k >= 1) is named model k + offset in refusals (nam_b200_bank_add_models checks its
// documents against model 0 under the indices they would receive)
BankCheck check_bank(const std::vector<ModelSpec>& specs, int offset = 0)
{
  BankCheck r;
  auto index = [&](size_t k) { return k == 0 ? 0 : (int)k + offset; };
  auto refuse = [&](int code, const std::string& why) {
    r.code = code;
    r.reason = why;
    return r;
  };
  if (specs.empty())
    return refuse(NAM_B200_ERR_INVALID_ARGUMENT, "n_models must be >= 1");
  if (specs[0].arch == Arch::LSTM)
  {
    r.family = KernelFamily::Lstm;
    for (size_t k = 0; k < specs.size(); k++)
    {
      const std::string mk = "model " + std::to_string(index(k)) + ": ";
      if (specs[k].arch != Arch::LSTM)
        return refuse(NAM_B200_ERR_UNSUPPORTED, mk + "architecture " + specs[k].architecture
                                                  + ": a bank's models share model 0's architecture (LSTM)");
      const std::string why = lstm_refusal(specs[k]); // (what an ordinary handle of the model would refuse)
      if (!why.empty())
        return refuse(NAM_B200_ERR_UNSUPPORTED, mk + why);
    }
    for (size_t k = 1; k < specs.size(); k++)
    {
      const std::string d = lstm_bank_difference(index(k), specs[k], specs[0]);
      if (!d.empty())
        return refuse(NAM_B200_ERR_MODEL, d);
    }
    return r;
  }
  auto family_name = [](KernelFamily f) { return f == KernelFamily::Fused ? "fused" : "general"; };
  for (size_t k = 0; k < specs.size(); k++)
  {
    const ModelSpec& s = specs[k];
    const std::string mk = "model " + std::to_string(index(k)) + ": ";
    if (s.arch == Arch::Container)
      return refuse(NAM_B200_ERR_UNSUPPORTED, mk + "architecture: a slimmable document (SlimmableContainer or slimmable "
                                                   "WaveNet); a bank serves plain WaveNets, ConvNets and LSTMs");
    if (s.arch != Arch::WaveNet && s.arch != Arch::ConvNet && s.arch != Arch::LSTM)
      return refuse(NAM_B200_ERR_UNSUPPORTED, mk + "architecture " + s.architecture
                                                + ": a bank serves WaveNets, ConvNets or LSTMs only");
    if (s.arch != specs[0].arch)
      return refuse(NAM_B200_ERR_UNSUPPORTED, mk + "architecture " + s.architecture
                                                + ": a bank's models share model 0's architecture (" + specs[0].architecture + ")");
    // the kernel an ordinary handle of the model gets by default, or its refusal
    KernelChoice c = choose_kernel(s, 0);
    if (c.code != NAM_B200_OK)
      return refuse(c.code, mk + (s.arch == Arch::WaveNet ? "kernel: " : "") + c.refusal);
    if (k == 0)
      r.family = c.family;
    else if (c.family != r.family)
      return refuse(NAM_B200_ERR_UNSUPPORTED,
                    mk + "kernel: served by the " + family_name(c.family) + " kernel"
                      + (c.family == KernelFamily::General ? " (fused kernel: " + c.plan.why_not + ")" : std::string())
                      + "; model 0 (" + family_name(r.family) + " family) chooses the bank's kernel family");
    if (c.family == KernelFamily::Fused)
      r.plans.push_back(std::move(c.plan));
    else
      r.gplans.push_back(std::move(c.gplan));
  }
  for (size_t k = 1; k < specs.size(); k++)
  {
    const std::string d = r.family == KernelFamily::Fused
                            ? bank_difference(index(k), specs[k], r.plans[k], specs[0], r.plans[0])
                            : general_bank_difference(index(k), specs[k], r.gplans[k], specs[0], r.gplans[0]);
    if (!d.empty())
      return refuse(NAM_B200_ERR_MODEL, d);
  }
  return r;
}

// Model i of a checked list as the bank stores it: the fused family's packed blob (its output scale goes to d_head_scales),
// an LSTM's weights, or the general kernel's weights -- a general WaveNet's followed by its net and condition_dsp output
// scales, which the BANK instantiation reads from the blob (float4 loads of every blob)
std::vector<float> bank_blob(const BankCheck& bc, const std::vector<ModelSpec>& specs, size_t i)
{
  if (bc.family == KernelFamily::Lstm)
    return lstm_blob(specs[i]);
  if (bc.family == KernelFamily::Fused)
    return bc.plans[i].blob;
  const GenericPlan& gp = bc.gplans[i];
  std::vector<float> b = gp.weights;
  if (specs[i].arch == Arch::WaveNet)
    b.insert(b.end(), {gp.net.head_scale, gp.cond.head_scale});
  return b;
}

// specs[i0 ..] (checked in bc) become models k0 .. of the bank: their blobs, output scales and record headers, queued on
// the handle's stream (the host sources are pageable: each copy stages them before returning).  The caller orders these
// writes after every reader of the slots they overwrite.
void upload_bank_models(nam_b200_model* m, const std::vector<ModelSpec>& specs, const BankCheck& bc, size_t i0, int k0)
{
  const size_t n = specs.size() - i0, stride = (size_t)m->weight_stride;
  std::vector<float> blobs(n * stride, 0.0f), scales(n, 0.0f);
  std::vector<StateRecordHeader> headers(n);
  for (size_t i = 0; i < n; i++)
  {
    const std::vector<float> blob = bank_blob(bc, specs, i0 + i);
    std::copy(blob.begin(), blob.end(), blobs.begin() + i * stride);
    if (bc.family == KernelFamily::Fused)
      scales[i] = bc.plans[i0 + i].head_scale;
    headers[i] = state_record_header(specs[i0 + i], m->record_floats);
  }
  CUDA_CHECK(cudaMemcpyAsync(m->d_weights + (size_t)k0 * stride, blobs.data(), blobs.size() * sizeof(float),
                             cudaMemcpyHostToDevice, m->stream));
  if (m->d_head_scales)
    CUDA_CHECK(cudaMemcpyAsync(m->d_head_scales + k0, scales.data(), n * sizeof(float), cudaMemcpyHostToDevice, m->stream));
  if (m->state_error.empty())
  {
    CUDA_CHECK(cudaMemcpyAsync(reinterpret_cast<unsigned char*>(m->d_bank_headers) + (size_t)k0 * kStateHeaderBytes,
                               headers.data(), n * kStateHeaderBytes, cudaMemcpyHostToDevice, m->stream));
    m->bank_headers.resize(std::max(m->bank_headers.size(), (size_t)k0 + n));
    std::copy(headers.begin(), headers.end(), m->bank_headers.begin() + k0);
  }
}

// A bank handle: an ordinary handle of model 0 on the precompiled kernels, then the blobs, output scales (WaveNet), record
// headers and model rows of `capacity` models, the first K of them filled
void setup_bank(nam_b200_model* m, std::vector<ModelSpec>&& specs, const BankCheck& bc, int capacity)
{
  const int K = (int)specs.size();
  const bool lstm = bc.family == KernelFamily::Lstm, fused = bc.family == KernelFamily::Fused;
  m->is_bank = true;
  m->bank_size = K;
  m->bank_capacity = capacity;
  m->weight_stride = (long)((bank_blob(bc, specs, 0).size() + 3) & ~(size_t)3);
  CUDA_CHECK(cudaFree(m->d_weights));
  m->d_weights = nullptr;
  CUDA_CHECK(cudaMalloc(&m->d_weights, (size_t)capacity * m->weight_stride * sizeof(float)));
  if (fused)
    CUDA_CHECK(cudaMalloc(&m->d_head_scales, (size_t)capacity * sizeof(float)));
  if (m->state_error.empty())
    CUDA_CHECK(cudaMalloc(&m->d_bank_headers, (size_t)capacity * kStateHeaderBytes));
  // the model rows behind the streams' rows
  CUDA_CHECK(cudaFree(m->d_state));
  m->d_state = nullptr;
  CUDA_CHECK(cudaMalloc(&m->d_state, (size_t)m->state_stride * state_rows(m) * sizeof(float)));
  // slot tables of up to max(max_batch, capacity) positions (prewarm_bank runs the model rows in one launch); an LSTM
  // bank's Reset runs the streams and the model rows in one launch
  const size_t n_slots = lstm ? (size_t)m->opts.max_batch + capacity : (size_t)std::max(m->opts.max_batch, capacity);
  m->h_slots.assign(n_slots, StreamRef{0, 0u, 0, 0});
  CUDA_CHECK(cudaFree(m->d_slots));
  m->d_slots = nullptr;
  CUDA_CHECK(cudaMalloc(&m->d_slots, n_slots * sizeof(StreamRef)));
  upload_bank_models(m, specs, bc, 0, 0);
  m->bank_specs = std::move(specs);
  m->spec_state = 0;
  m->spec_note = "model bank of up to " + std::to_string(capacity) + " models: the precompiled kernels, which read each "
                 "stream's weights as data (a model-specialised kernel compiles one model's weights into its code)";
  if (bc.family == KernelFamily::General)
    setup_generic_bank_kernel(m); // (throws under jit = 1 when the shape-compiled kernel cannot be had)
  init_state(m);
  CUDA_CHECK(cudaStreamSynchronize(m->stream));
}

// nam_b200_options::bank_capacity of a bank of n_models documents (0 = n_models), or the refusal
int bank_capacity_option(const nam_b200_options* opts, int n_models, int* capacity)
{
  const bool has = opts && (size_t)std::max(opts->struct_size, 0) >= offsetof(nam_b200_options, bank_capacity) + sizeof(int32_t);
  const int c = has ? opts->bank_capacity : 0;
  if (c < 0 || (c > 0 && c < n_models))
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "model bank: bank_capacity = " + std::to_string(c) + " must be 0 (the number of "
                                                 "documents) or >= n_models = " + std::to_string(n_models));
  *capacity = std::max(c, n_models);
  return NAM_B200_OK;
}

// Documents -> the specs of a bank's models; "model k" in a refusal is first + i for texts[i]
int bank_specs_from_texts(const char* const* texts, int n, int first, bool fast_tanh, const std::string& what,
                          std::vector<ModelSpec>* specs)
{
  LoadOptions lo;
  lo.fast_tanh = fast_tanh;
  for (int i = 0; i < n; i++)
  {
    const std::string mk = what + "model " + std::to_string(first + i) + ": ";
    if (!texts[i])
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, mk + "null document");
    try
    {
      specs->push_back(model_spec_from_text(texts[i], lo));
    }
    catch (const json::ParseError& ex)
    {
      return fail(NAM_B200_ERR_FILE, mk + ex.what());
    }
    catch (const std::exception& ex)
    {
      return fail(NAM_B200_ERR_MODEL, mk + ex.what());
    }
  }
  return NAM_B200_OK;
}

int create_bank(std::vector<ModelSpec>&& specs, const nam_b200_options* user_opts, int capacity, nam_b200_model** out)
{
  const BankCheck bc = check_bank(specs);
  if (bc.code != NAM_B200_OK)
    return fail(bc.code, "model bank: " + bc.reason);
  nam_b200_options o;
  nam_b200_default_options(&o);
  if (user_opts)
  {
    std::memcpy(&o, user_opts, std::min<size_t>(sizeof o, (size_t)std::max(user_opts->struct_size, 0)));
    o.struct_size = sizeof o;
  }
  if (o.jit == 1 && (bc.family == KernelFamily::Fused || bc.family == KernelFamily::Lstm))
    return fail(NAM_B200_ERR_UNSUPPORTED, "model bank: jit = 1 (required) cannot be met: a model-specialised kernel compiles "
                                          "one model's weights into its code, a bank's streams each bring their own");
  if (o.kernel_geometry == 4 && (bc.family == KernelFamily::Fused || bc.family == KernelFamily::Lstm))
    return fail(NAM_B200_ERR_UNSUPPORTED, "model bank: kernel_geometry 4 (the general kernel) does not take banks of the fused "
                                          "WaveNet or LSTM families (model 0 chooses the family)");
  // Fused and LSTM banks: jit 0 / 3 run the precompiled kernels, silently (nam_b200_jit_note says why).  General banks: model
  // 0's handle is made without its model-specialised kernel, then setup_bank applies the requested jit to the kernel compiled
  // for the bank's shape.  ConvNet banks take jit as an ordinary ConvNet handle does (it has no compiled kernel).
  const int user_jit = o.jit;
  if (bc.family != KernelFamily::ConvNet)
    o.jit = 2;
  if (bc.family == KernelFamily::General && o.kernel_geometry != 0)
    o.kernel_geometry = 4; // (the general kernel is the family's: a fused geometry must not move model 0 onto the fused kernel)
  nam_b200_model* h = nullptr;
  const int rc = create_common(ModelSpec(specs[0]), &o, &h);
  if (rc != NAM_B200_OK)
    return rc;
  std::unique_ptr<nam_b200_model> m(h);
  if (bc.family == KernelFamily::General)
    m->opts.jit = user_jit;
  const int rc2 = guarded(m.get(), [&]() -> int {
    setup_bank(m.get(), std::move(specs), bc, capacity);
    return NAM_B200_OK;
  });
  if (rc2 == NAM_B200_OK)
    *out = m.release();
  return rc2;
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
  // what a handle with the default options runs
  const KernelChoice c = choose_kernel(spec, 0);
  static const char* const kernel_names[] = {"fused", "generic", "convnet", "lstm", "linear"};
  const bool ok = c.code == NAM_B200_OK;
  const char* kernel = ok ? kernel_names[(int)c.family] : "unsupported";
  std::string reason = !ok ? c.refusal : (c.family == KernelFamily::General ? "fused kernel: " + c.plan.why_not : "");
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
                spec.sample_rate, c.flops_per_frame, c.state_stride * 4, kernel, c.variant, spec.loudness ? "true" : "false",
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
    // the kernel a handle with the default options looks for (a WaveNet create refuses: its general kernel's refusal)
    const KernelChoice c = choose_kernel(ms, 0);
    const bool fused_family = ms.arch == Arch::WaveNet && c.code == NAM_B200_OK && c.family == KernelFamily::Fused;
    SpecBuild b = ms.arch == Arch::LSTM ? build_lstm_spec_kernel(ms)
                  : fused_family        ? build_spec_kernel(c.plan, spec_geometry_for(std::max(max_batch, 1), 132)) // H100 SXM
                                        : build_generic_spec_kernel(c.gplan);
    // WaveNets: also the low-latency kernel for 64-frame calls (the plugin protocol), so that a first Reset finds it cached
    SpecBuild lat;
    if (fused_family)
      lat = build_lat_kernel(c.plan, 2);
    std::string why;
    for (char c : b.why_not.substr(0, 600))
      why += (c == '"' || c == '\\') ? '\'' : (c == '\n' ? ' ' : c);
    char buf[1024];
    std::snprintf(buf, sizeof buf,
                  "{\"ok\": %s, \"from_cache\": %s, \"compile_seconds\": %.3f, \"cubin_bytes\": %zu, \"threads\": %d, "
                  "\"frames_per_thread\": 1, \"smem_bytes\": %zu, \"why_not\": \"%s\", \"lat_ok\": %s, "
                  "\"lat_compile_seconds\": %.3f, \"lat_cubin_bytes\": %zu}",
                  b.ok ? "true" : "false", b.from_cache ? "true" : "false", b.compile_seconds, b.cubin.size() + b.cubin_extra.size(), b.geom.nt,
                  b.ok ? b.smem_bytes() : (size_t)0, why.c_str(), lat.ok ? "true" : "false", lat.compile_seconds,
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

// the handle's info with the document-level fields (loudness, levels, sample rate, weights) of `spec`
static int fill_info(const nam_b200_model* m, const ModelSpec& spec, nam_b200_info* info)
{
  nam_b200_info r;
  std::memset(&r, 0, sizeof(r));
  r.struct_size = sizeof(nam_b200_info);
  r.architecture = (int)spec.arch;
  r.in_channels = spec.in_channels;
  r.out_channels = spec.out_channels;
  r.prewarm_samples = spec.prewarm_samples;
  r.max_batch = m->opts.max_batch;
  r.max_frames = call_max_frames(m);
  r.has_loudness = spec.loudness.has_value();
  r.has_input_level = spec.input_level.has_value();
  r.has_output_level = spec.output_level.has_value();
  r.expected_sample_rate = spec.sample_rate;
  r.loudness = spec.loudness.value_or(0.0);
  r.input_level_dbu = spec.input_level.value_or(0.0);
  r.output_level_dbu = spec.output_level.value_or(0.0);
  r.n_weights = (int64_t)spec.n_weights;
  r.state_bytes_per_stream = (int64_t)m->state_stride * 4;
  r.flops_per_frame = m->flops_per_frame;
  r.kernel_variant = m->variant;
  r.jit_state = m->spec_state;
  r.jit_lat_state = m->lat_state;
  r.resample_up = m->rs.active ? m->rs.design.L : 1;
  r.resample_down = m->rs.active ? m->rs.design.M : 1;
  r.resample_latency_frames = m->rs.active ? (int32_t)std::lround(m->rs.design.latency_frames) : 0;
  const size_t n = std::min<size_t>(sizeof(r), (size_t)std::max(info->struct_size, 0));
  const int32_t user_size = info->struct_size;
  std::memcpy(info, &r, n);
  info->struct_size = user_size;
  return NAM_B200_OK;
}

int nam_b200_get_info(const nam_b200_model* m, nam_b200_info* info)
{
  m = active_model(m);
  if (!m || !info)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument");
  return fill_info(m, model_spec(m, 0), info); // (a bank: model 0's document, which nam_b200_bank_replace_model may change)
}

int nam_b200_reset(nam_b200_model* m, double sample_rate, int max_frames)
{
  // like the reference, the external rate is recorded but does not change the model's arithmetic (options.resample
  // converts to the model's rate around it)
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
    ResamplerDesign rd;
    bool convert = false;
    const std::string refusal = resampler_for(m, sample_rate, &rd, &convert);
    if (!refusal.empty())
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, refusal);
    setup_resampler(m, convert, rd, max_frames); // (m->max_frames: the model's maxBufferSize)
    const size_t ch = (size_t)std::max(m->spec.in_channels, m->spec.out_channels);
    ensure_staging(m, (size_t)m->opts.max_batch * staging_frames(m) * ch);
    ensure_pinned(m, (size_t)2 * staging_frames(m) * ch);
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
    if (m->is_bank && m->spec.arch == Arch::LSTM)
      prewarm_lstm_bank(m, true); // (also rebuilds the model rows when prewarm_on_reset = 0: h0 / c0)
    else if (m->opts.prewarm_on_reset)
      (m->is_bank ? prewarm_bank : prewarm)(m);
    CUDA_CHECK(cudaEventRecord(m->ev1, m->stream));
    // every stream is now in the state of a freshly reset one: keep stream 0's record for nam_b200_reset_streams (an LSTM
    // keeps its running state across a Reset, so its streams are re-derived per call instead; a bank keeps model rows)
    if (m->spec.arch != Arch::LSTM && m->state_error.empty() && !m->is_bank)
    {
      const int32_t s0 = 0;
      export_records(m, &s0, 1, m->d_fresh, 0, m->stream);
    }
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

// ---- per-stream state control ---------------------------------------------------------------------------------------
int64_t nam_b200_stream_state_size(const nam_b200_model* m)
{
  m = active_model(m);
  if (!m)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null model handle");
  if (!m->state_error.empty())
    return fail(NAM_B200_ERR_UNSUPPORTED, "no per-stream state records for this handle: " + m->state_error);
  return (int64_t)record_bytes(m);
}

int nam_b200_reset_streams(nam_b200_model* m, const int32_t* streams, int n, int fresh)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    int rc = check_state_calls(m, "reset_streams");
    if (rc == NAM_B200_OK)
      rc = check_stream_list(m, streams, n, "streams", true);
    if (rc != NAM_B200_OK || n == 0)
      return rc;
    if (m->spec.arch == Arch::LSTM && !(m->is_bank && fresh))
      lstm_reset_rows(m, streams, n, fresh != 0);
    else if (m->is_bank)
      bank_fan_out(m, streams, n, m->stream); // each stream's own model's fresh row
    else
      import_records(m, streams, n, m->d_fresh, 0, m->stream); // (fresh or not: Reset forgets the past)
    rs_zero(m, streams, n, m->stream);
    CUDA_CHECK(cudaStreamSynchronize(m->stream));
    return NAM_B200_OK;
  });
}

int nam_b200_copy_streams(nam_b200_model* m, const int32_t* src, const int32_t* dst, int n)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    int rc = check_state_calls(m, "copy_streams");
    if (rc == NAM_B200_OK)
      rc = check_stream_list(m, src, n, "src", false);
    if (rc == NAM_B200_OK)
      rc = check_stream_list(m, dst, n, "dst", true);
    if (rc != NAM_B200_OK || n == 0)
      return rc;
    // gather every source row into scratch, then scatter: overlapping lists (a swap) see the sources as they were
    const size_t rows = (size_t)n * (size_t)m->state_stride;
    const bool linear = m->spec.arch == Arch::Linear && m->d_state_tmp;
    ensure_xfer(m, rows * sizeof(float) * (linear ? 2 : 1));
    std::vector<StreamRef> refs((size_t)2 * n);
    for (int i = 0; i < n; i++)
    {
      refs[(size_t)i] = StreamRef{src[i], 0, 0, 0};
      refs[(size_t)(n + i)] = StreamRef{dst[i], 0, 0, 0};
    }
    const StreamRef* d_refs = upload_refs(m, refs, m->stream);
    float* scratch = reinterpret_cast<float*>(m->d_xfer);
    copy_rows(m, scratch, nullptr, m->d_state, d_refs, n, m->stream);
    copy_rows(m, m->d_state, d_refs + n, scratch, nullptr, n, m->stream);
    if (linear) // both buffers of the double buffer; the destination keeps the source's buffer parity
    {
      copy_rows(m, scratch + rows, nullptr, m->d_state_tmp, d_refs, n, m->stream);
      copy_rows(m, m->d_state_tmp, d_refs + n, scratch + rows, nullptr, n, m->stream);
    }
    std::vector<uint32_t> clock((size_t)n), flips((size_t)n);
    std::vector<int32_t> model((size_t)n); // (a bank: the destination takes the source's model along with its state)
    for (int i = 0; i < n; i++)
    {
      clock[(size_t)i] = m->stream_clock[(size_t)src[i]];
      flips[(size_t)i] = m->stream_flips[(size_t)src[i]];
      model[(size_t)i] = m->stream_model[(size_t)src[i]];
    }
    for (int i = 0; i < n; i++)
    {
      m->stream_clock[(size_t)dst[i]] = clock[(size_t)i];
      m->stream_flips[(size_t)dst[i]] = flips[(size_t)i];
      m->stream_model[(size_t)dst[i]] = model[(size_t)i];
    }
    rs_copy(m, src, dst, n, m->stream);
    m->streams_identical = false;
    recount_phase(m);
    CUDA_CHECK(cudaStreamSynchronize(m->stream));
    return NAM_B200_OK;
  });
}

int nam_b200_export_streams(nam_b200_model* m, const int32_t* streams, int n, void* dst, int64_t record_stride)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    int rc = check_state_calls(m, "export_streams");
    if (rc == NAM_B200_OK)
      rc = check_stream_list(m, streams, n, "streams", false);
    if (rc == NAM_B200_OK)
      rc = check_records(m, dst, n, record_stride, false);
    if (rc != NAM_B200_OK || n == 0)
      return rc;
    const size_t rb = record_bytes(m);
    const int group = (int)std::max<size_t>(1, kRecordStagingBytes / rb);
    ensure_xfer(m, (size_t)std::min(n, group) * rb);
    for (int i0 = 0; i0 < n; i0 += group)
    {
      const int k = std::min(group, n - i0);
      export_records(m, streams + i0, k, m->d_xfer, (long)rb, m->stream);
      rs_export(m, streams + i0, k, m->d_xfer, (long)rb, m->stream);
      CUDA_CHECK(cudaMemcpy2DAsync(static_cast<unsigned char*>(dst) + (size_t)i0 * record_stride, (size_t)record_stride, m->d_xfer,
                                   rb, rb, (size_t)k, cudaMemcpyDeviceToHost, m->stream));
      CUDA_CHECK(cudaStreamSynchronize(m->stream));
    }
    return NAM_B200_OK;
  });
}

int nam_b200_import_streams(nam_b200_model* m, const int32_t* streams, int n, const void* src, int64_t record_stride)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    int rc = check_state_calls(m, "import_streams");
    if (rc == NAM_B200_OK)
      rc = check_stream_list(m, streams, n, "streams", true);
    if (rc == NAM_B200_OK)
      rc = check_records(m, src, n, record_stride, false, true);
    std::vector<int> model((size_t)std::max(n, 0));
    for (int i = 0; i < n && rc == NAM_B200_OK; i++)
      rc = check_record_header(m, static_cast<const unsigned char*>(src) + (size_t)i * record_stride, i, streams[i], &model[(size_t)i]);
    std::vector<uint32_t> phases;
    if (rc == NAM_B200_OK && m->rs.active)
    {
      std::vector<float> v((size_t)n);
      const size_t at = kStateHeaderBytes + 4 * (size_t)(m->record_floats + rs_record_floats(m) - 1);
      for (int i = 0; i < n; i++)
        std::memcpy(&v[(size_t)i], static_cast<const unsigned char*>(src) + (size_t)i * record_stride + at, 4);
      rc = rs_record_phases(m, streams, v.data(), n, &phases);
    }
    if (rc != NAM_B200_OK || n == 0)
      return rc;
    for (int i = 0; i < n; i++) // (a bank: the stream runs the record's model from now on)
      m->stream_model[(size_t)streams[i]] = model[(size_t)i];
    const size_t rb = record_bytes(m);
    const int group = (int)std::max<size_t>(1, kRecordStagingBytes / rb);
    ensure_xfer(m, (size_t)std::min(n, group) * rb);
    for (int i0 = 0; i0 < n; i0 += group)
    {
      const int k = std::min(group, n - i0);
      CUDA_CHECK(cudaMemcpy2DAsync(m->d_xfer, rb, static_cast<const unsigned char*>(src) + (size_t)i0 * record_stride,
                                   (size_t)record_stride, rb, (size_t)k, cudaMemcpyHostToDevice, m->stream));
      import_records(m, streams + i0, k, m->d_xfer, (long)rb, m->stream);
      rs_import(m, streams + i0, k, m->d_xfer, (long)rb, phases.data() + i0, m->stream);
      CUDA_CHECK(cudaStreamSynchronize(m->stream));
    }
    return NAM_B200_OK;
  });
}

int nam_b200_export_streams_device(nam_b200_model* m, const int32_t* streams, int n, void* dst_device, int64_t record_stride,
                                   void* cuda_stream)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    int rc = check_state_calls(m, "export_streams_device");
    if (rc == NAM_B200_OK)
      rc = check_stream_list(m, streams, n, "streams", false);
    if (rc == NAM_B200_OK)
      rc = check_records(m, dst_device, n, record_stride, true);
    if (rc != NAM_B200_OK || n == 0)
      return rc;
    const cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : m->stream;
    export_records(m, streams, n, static_cast<unsigned char*>(dst_device), (long)record_stride, st);
    rs_export(m, streams, n, static_cast<unsigned char*>(dst_device), (long)record_stride, st);
    return NAM_B200_OK;
  });
}

int nam_b200_import_streams_device(nam_b200_model* m, const int32_t* streams, int n, const void* src_device,
                                   int64_t record_stride, void* cuda_stream)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    int rc = check_state_calls(m, "import_streams_device");
    if (rc == NAM_B200_OK)
      rc = check_stream_list(m, streams, n, "streams", true);
    if (rc == NAM_B200_OK)
      rc = check_records(m, src_device, n, record_stride, true, true);
    if (rc != NAM_B200_OK || n == 0)
      return rc;
    const cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : m->stream;
    // the headers come to the host and are checked before anything is launched
    std::vector<unsigned char> headers((size_t)n * kStateHeaderBytes);
    CUDA_CHECK(cudaMemcpy2DAsync(headers.data(), kStateHeaderBytes, src_device, (size_t)record_stride, kStateHeaderBytes, (size_t)n,
                                 cudaMemcpyDeviceToHost, st));
    std::vector<float> phase_values((size_t)n); // (a converting handle: each record's resample_phase, the payload's last float)
    if (m->rs.active)
      CUDA_CHECK(cudaMemcpy2DAsync(phase_values.data(), 4,
                                   static_cast<const unsigned char*>(src_device) + kStateHeaderBytes
                                     + 4 * (size_t)(m->record_floats + rs_record_floats(m) - 1),
                                   (size_t)record_stride, 4, (size_t)n, cudaMemcpyDeviceToHost, st));
    CUDA_CHECK(cudaStreamSynchronize(st));
    std::vector<int> model((size_t)n);
    for (int i = 0; i < n; i++)
    {
      rc = check_record_header(m, headers.data() + (size_t)i * kStateHeaderBytes, i, streams[i], &model[(size_t)i]);
      if (rc != NAM_B200_OK)
        return rc;
    }
    std::vector<uint32_t> phases;
    if (m->rs.active && (rc = rs_record_phases(m, streams, phase_values.data(), n, &phases)) != NAM_B200_OK)
      return rc;
    for (int i = 0; i < n; i++)
      m->stream_model[(size_t)streams[i]] = model[(size_t)i];
    import_records(m, streams, n, static_cast<const unsigned char*>(src_device), (long)record_stride, st);
    rs_import(m, streams, n, static_cast<const unsigned char*>(src_device), (long)record_stride, phases.data(), st);
    return NAM_B200_OK;
  });
}

int nam_b200_resampler_json(double host_rate, double model_rate, char* out, int64_t capacity)
{
  if (!out || capacity < 1)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null or empty output buffer");
  ResamplerDesign d;
  std::string why;
  if (!design_resampler(host_rate, model_rate, &d, &why))
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, why);
  const std::string js = resampler_json(d);
  if ((int64_t)js.size() >= capacity)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "output buffer too small: " + std::to_string(js.size() + 1) + " bytes needed");
  std::memcpy(out, js.c_str(), js.size() + 1);
  return NAM_B200_OK;
}

int nam_b200_state_layout_json(const char* nam_json_text, char* out, int64_t capacity)
{
  if (!nam_json_text || !out || capacity <= 0)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument or empty output buffer");
  try
  {
    LoadOptions lo;
    ModelSpec ms = model_spec_from_text(nam_json_text, lo);
    if (ms.arch == Arch::Container) // the default (largest) sub-model, the one a new handle serves
      ms = model_spec_from_text(ms.submodels.back().model_json, lo);
    const std::string s = state_layout_json(ms);
    if ((int64_t)s.size() >= capacity)
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, "the state layout needs " + std::to_string(s.size() + 1) + " bytes, the buffer has "
                                                   + std::to_string(capacity));
    std::memcpy(out, s.c_str(), s.size() + 1);
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

// ---- model banks ---------------------------------------------------------------------------------------------------------
int nam_b200_create_bank_from_json(const char* const* texts, int n_models, const nam_b200_options* opts, nam_b200_model** out)
{
  if (!out)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  if (n_models < 1)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "model bank: n_models = " + std::to_string(n_models) + " must be >= 1");
  if (!texts)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "model bank: null document list");
  int capacity = 0;
  if (const int rc = bank_capacity_option(opts, n_models, &capacity); rc != NAM_B200_OK)
    return rc;
  if (capacity == 1) // (a bank that can only ever hold its one document is the ordinary handle)
    return nam_b200_create_from_json(texts[0], opts, out);
  std::vector<ModelSpec> specs;
  if (const int rc = bank_specs_from_texts(texts, n_models, 0, opts && opts->fast_tanh != 0, "model bank: ", &specs);
      rc != NAM_B200_OK)
    return rc;
  return create_bank(std::move(specs), opts, capacity, out);
}

int nam_b200_create_bank_from_files(const char* const* paths, int n_models, const nam_b200_options* opts, nam_b200_model** out)
{
  if (!out)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  if (n_models < 1)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "model bank: n_models = " + std::to_string(n_models) + " must be >= 1");
  if (!paths)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "model bank: null path list");
  int capacity = 0;
  if (const int rc = bank_capacity_option(opts, n_models, &capacity); rc != NAM_B200_OK)
    return rc;
  if (capacity == 1)
    return nam_b200_create_from_file(paths[0], opts, out);
  LoadOptions lo;
  lo.fast_tanh = opts ? (opts->fast_tanh != 0) : false;
  std::vector<ModelSpec> specs;
  for (int k = 0; k < n_models; k++)
  {
    const std::string mk = "model bank: model " + std::to_string(k) + ": ";
    if (!paths[k])
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, mk + "null path");
    try
    {
      specs.push_back(model_spec_from_file(paths[k], lo));
    }
    catch (const NamFileValidationError& ex)
    {
      return fail(NAM_B200_ERR_FILE, mk + ex.what());
    }
    catch (const std::exception& ex)
    {
      return fail(NAM_B200_ERR_MODEL, mk + ex.what());
    }
  }
  return create_bank(std::move(specs), opts, capacity, out);
}

int nam_b200_bank_check_json(const char* const* texts, int n_models, char* out, int64_t capacity)
{
  if (!out || capacity <= 0)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument or empty output buffer");
  std::string reason;
  std::vector<ModelSpec> specs;
  if (n_models < 1)
    reason = "n_models = " + std::to_string(n_models) + " must be >= 1";
  else if (!texts)
    reason = "null document list";
  for (int k = 0; reason.empty() && k < n_models; k++)
  {
    try
    {
      if (!texts[k])
        throw std::runtime_error("null document");
      specs.push_back(model_spec_from_text(texts[k], LoadOptions{}));
    }
    catch (const std::exception& ex)
    {
      reason = "model " + std::to_string(k) + ": " + ex.what();
    }
  }
  if (reason.empty())
    reason = check_bank(specs).reason;
  for (auto& ch : reason)
    if (ch == '"' || ch == '\\' || ch == '\n')
      ch = ' ';
  std::string s = std::string("{\"ok\": ") + (reason.empty() ? "true" : "false") + ", \"n_models\": " + std::to_string(n_models)
                  + ", \"reason\": \"" + reason + "\", \"fingerprints\": [";
  for (size_t k = 0; k < specs.size(); k++) // (as nam_b200_state_layout_json writes them)
    s += std::string(k ? ", " : "") + std::to_string((unsigned long long)specs[k].fingerprint);
  s += "]}";
  if ((int64_t)s.size() >= capacity)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "the bank check needs " + std::to_string(s.size() + 1) + " bytes, the buffer has "
                                                 + std::to_string(capacity));
  std::memcpy(out, s.c_str(), s.size() + 1);
  return NAM_B200_OK;
}

int nam_b200_bank_jit_prepare_json(const char* const* texts, int n_models, int fast_tanh, char* out, int64_t capacity)
{
  if (!out || capacity <= 0 || !texts || n_models < 1)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument, empty output buffer or n_models < 1");
  LoadOptions lo;
  lo.fast_tanh = fast_tanh != 0;
  std::vector<ModelSpec> specs;
  try
  {
    for (int k = 0; k < n_models; k++)
    {
      if (!texts[k])
        throw std::runtime_error("model " + std::to_string(k) + ": null document");
      specs.push_back(model_spec_from_text(texts[k], lo));
    }
  }
  catch (const std::exception& ex)
  {
    return fail(NAM_B200_ERR_MODEL, ex.what());
  }
  const BankCheck bc = check_bank(specs);
  if (bc.code != NAM_B200_OK)
    return fail(bc.code, "model bank: " + bc.reason);
  if (bc.family != KernelFamily::General)
    return fail(NAM_B200_ERR_UNSUPPORTED, "model bank: only banks of general-kernel WaveNets have a shape-compiled kernel");
  const SpecBuild b = build_generic_spec_kernel(bc.gplans[0], true);
  std::string why;
  for (char c : b.why_not.substr(0, 600))
    why += (c == '"' || c == '\\') ? '\'' : (c == '\n' ? ' ' : c);
  char buf[1024];
  std::snprintf(buf, sizeof buf,
                "{\"ok\": %s, \"from_cache\": %s, \"compile_seconds\": %.3f, \"cubin_bytes\": %zu, \"threads\": %d, "
                "\"smem_bytes\": %zu, \"why_not\": \"%s\"}",
                b.ok ? "true" : "false", b.from_cache ? "true" : "false", b.compile_seconds, b.cubin.size(), kGenTile,
                generic_bank_blob_floats(bc.gplans[0]) * sizeof(float), why.c_str());
  const std::string s(buf);
  if ((int64_t)s.size() >= capacity)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "the report needs " + std::to_string(s.size() + 1) + " bytes");
  std::memcpy(out, s.c_str(), s.size() + 1);
  return NAM_B200_OK;
}

int nam_b200_bank_size(const nam_b200_model* m)
{
  m = active_model(m);
  if (!m)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null model handle");
  return m->bank_size;
}

int nam_b200_bank_capacity(const nam_b200_model* m)
{
  m = active_model(m);
  if (!m)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null model handle");
  return m->bank_capacity;
}

int nam_b200_bank_add_models(nam_b200_model* m, const char* const* texts, int n, int32_t* first_index)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    if (!texts || !first_index)
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, "bank_add_models: null argument");
    if (n < 1)
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, "bank_add_models: n = " + std::to_string(n) + " must be >= 1");
    const int K = m->bank_size;
    if (n > m->bank_capacity - K)
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, "bank_add_models: " + std::to_string(n) + " documents do not fit: the bank holds "
                                                   + std::to_string(K) + " of its bank_capacity = " + std::to_string(m->bank_capacity)
                                                   + " models");
    // every document is checked against model 0 before anything changes: a refusal leaves the handle as it was
    std::vector<ModelSpec> specs{m->bank_specs[0]};
    int rc = bank_specs_from_texts(texts, n, K, m->opts.fast_tanh != 0, "bank_add_models: ", &specs);
    if (rc != NAM_B200_OK)
      return rc;
    const BankCheck bc = check_bank(specs, K - 1);
    if (bc.code != NAM_B200_OK)
      return fail(bc.code, "model bank: " + bc.reason);
    // (slots K .. K + n - 1 are read by no call yet)
    upload_bank_models(m, specs, bc, 1, K);
    m->bank_specs.insert(m->bank_specs.end(), std::make_move_iterator(specs.begin() + 1), std::make_move_iterator(specs.end()));
    m->bank_size = K + n;
    if (m->is_reset)
      prepare_bank_rows(m, K, n); // (before the first reset, nam_b200_reset prepares them with the others)
    CUDA_CHECK(cudaStreamSynchronize(m->stream));
    *first_index = K;
    return NAM_B200_OK;
  });
}

int nam_b200_bank_replace_model(nam_b200_model* m, int k, const char* text)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    if (!m->is_bank)
      return fail(NAM_B200_ERR_UNSUPPORTED, "bank_replace_model: not a model bank (create one with nam_b200_create_bank_*)");
    if (k < 0 || k >= m->bank_size)
      return fail(NAM_B200_ERR_INVALID_ARGUMENT, "bank_replace_model: model index " + std::to_string(k) + " outside [0, bank_size="
                                                   + std::to_string(m->bank_size) + ")");
    int bound = 0, lowest = -1;
    for (size_t s = 0; s < m->stream_model.size(); s++)
      if (m->stream_model[s] == k && bound++ == 0)
        lowest = (int)s;
    if (bound > 0)
      return fail(NAM_B200_ERR_STATE, "bank_replace_model: " + std::to_string(bound) + " stream(s) are bound to model "
                                        + std::to_string(k) + " (the lowest: stream " + std::to_string(lowest)
                                        + "); move them with assign_streams first");
    std::vector<ModelSpec> specs{m->bank_specs[0]};
    int rc = bank_specs_from_texts(&text, 1, k, m->opts.fast_tanh != 0, "bank_replace_model: ", &specs);
    if (rc != NAM_B200_OK)
      return rc;
    const BankCheck bc = check_bank(specs, k - 1);
    if (bc.code != NAM_B200_OK)
      return fail(bc.code, "model bank: " + bc.reason);
    // an earlier call of the handle, on any CUDA stream, may still read blob k or row k: every bank call carries a table,
    // so the last of them is marked by slots_free
    if (m->slots_used)
      CUDA_CHECK(cudaStreamWaitEvent(m->stream, m->slots_free, 0));
    upload_bank_models(m, specs, bc, 1, k);
    m->bank_specs[(size_t)k] = std::move(specs[1]);
    if (m->is_reset)
      prepare_bank_rows(m, k, 1);
    CUDA_CHECK(cudaStreamSynchronize(m->stream));
    return NAM_B200_OK;
  });
}

int nam_b200_assign_streams(nam_b200_model* m, const int32_t* streams, int n, const int32_t* models)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    int rc = check_state_calls(m, "assign_streams");
    if (rc == NAM_B200_OK)
      rc = check_stream_list(m, streams, n, "assign_streams: streams", true);
    if (rc == NAM_B200_OK && n > 0 && !models)
      rc = fail(NAM_B200_ERR_INVALID_ARGUMENT, "assign_streams: null model list");
    for (int i = 0; i < n && rc == NAM_B200_OK; i++)
      if (models[i] < 0 || models[i] >= m->bank_size)
        rc = fail(NAM_B200_ERR_INVALID_ARGUMENT, "assign_streams: models[" + std::to_string(i) + "] = " + std::to_string(models[i])
                                                   + ": model index outside [0, bank_size=" + std::to_string(m->bank_size) + ")");
    if (rc != NAM_B200_OK || n == 0)
      return rc;
    if (!m->is_bank)
      return nam_b200_reset_streams(m, streams, n, 0);
    for (int i = 0; i < n; i++)
      m->stream_model[(size_t)streams[i]] = models[i];
    bank_fan_out(m, streams, n, m->stream);
    rs_zero(m, streams, n, m->stream);
    CUDA_CHECK(cudaStreamSynchronize(m->stream));
    return NAM_B200_OK;
  });
}

int nam_b200_stream_models(const nam_b200_model* m, const int32_t* streams, int n, int32_t* out)
{
  m = active_model(m);
  if (!m)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null model handle");
  const int rc = check_stream_list(m, streams, n, "stream_models: streams", false);
  if (rc != NAM_B200_OK)
    return rc;
  if (n > 0 && !out)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "stream_models: null output");
  for (int i = 0; i < n; i++)
    out[i] = m->stream_model[(size_t)streams[i]];
  return NAM_B200_OK;
}

int nam_b200_bank_model_info(const nam_b200_model* m, int k, nam_b200_info* info)
{
  m = active_model(m);
  if (!m || !info)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT, "null argument");
  if (k < 0 || k >= m->bank_size)
    return fail(NAM_B200_ERR_INVALID_ARGUMENT,
                "bank_model_info: model index " + std::to_string(k) + " outside [0, bank_size=" + std::to_string(m->bank_size) + ")");
  return fill_info(m, model_spec(m, k), info);
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
    run_call(m, in_device, out_device, batch, n_frames, (long)in_stride, (long)out_stride, st);
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
    process_host(m, nullptr, batch, in, out, n_frames, in_stride, out_stride);
    return NAM_B200_OK;
  });
}

int nam_b200_process_streams_f32(nam_b200_model* m, const int32_t* streams, int n, const float* in, float* out, int n_frames,
                                 int64_t in_stride, int64_t out_stride)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    const int rc = check_process_streams_args(m, "process_streams_f32", streams, n, in, out, n_frames, in_stride, out_stride);
    if (rc != NAM_B200_OK || n == 0 || n_frames == 0)
      return rc;
    process_host(m, streams, n, in, out, n_frames, in_stride, out_stride);
    return NAM_B200_OK;
  });
}

int nam_b200_process_streams_f32_device(nam_b200_model* m, const int32_t* streams, int n, const float* in_device,
                                        float* out_device, int n_frames, int64_t in_stride, int64_t out_stride,
                                        void* cuda_stream)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    const int rc =
      check_process_streams_args(m, "process_streams_f32_device", streams, n, in_device, out_device, n_frames, in_stride, out_stride);
    if (rc != NAM_B200_OK || n == 0 || n_frames == 0)
      return rc;
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : m->stream;
    CUDA_CHECK(cudaEventRecord(m->ev0, st));
    run_call(m, in_device, out_device, n, n_frames, (long)in_stride, (long)out_stride, st, streams);
    CUDA_CHECK(cudaEventRecord(m->ev1, st));
    m->timing_valid = true;
    return NAM_B200_OK;
  });
}

int nam_b200_process_streams_ragged_f32(nam_b200_model* m, const int32_t* streams, int n, const int32_t* n_frames,
                                        const float* in, float* out, int64_t in_stride, int64_t out_stride)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    int n_max = 0;
    const int rc =
      check_ragged_args(m, "process_streams_ragged_f32", streams, n, n_frames, in, out, in_stride, out_stride, &n_max);
    if (rc != NAM_B200_OK || n == 0 || n_max == 0)
      return rc;
    process_host(m, streams, n, in, out, n_max, in_stride, out_stride, n_frames);
    return NAM_B200_OK;
  });
}

int nam_b200_process_streams_ragged_f32_device(nam_b200_model* m, const int32_t* streams, int n, const int32_t* n_frames,
                                               const float* in_device, float* out_device, int64_t in_stride,
                                               int64_t out_stride, void* cuda_stream)
{
  m = active_model(m);
  return guarded(m, [&]() -> int {
    int n_max = 0;
    const int rc = check_ragged_args(m, "process_streams_ragged_f32_device", streams, n, n_frames, in_device, out_device,
                                     in_stride, out_stride, &n_max);
    if (rc != NAM_B200_OK || n == 0 || n_max == 0)
      return rc;
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : m->stream;
    CUDA_CHECK(cudaEventRecord(m->ev0, st));
    run_call(m, in_device, out_device, n, n_max, (long)in_stride, (long)out_stride, st, streams, n_frames);
    CUDA_CHECK(cudaEventRecord(m->ev1, st));
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
  if (o.resample != 0)
    return fail(NAM_B200_ERR_UNSUPPORTED, "resample = " + std::to_string(o.resample)
                                            + ": multi-GPU handles do not convert sample rates (use one handle per GPU)");
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
