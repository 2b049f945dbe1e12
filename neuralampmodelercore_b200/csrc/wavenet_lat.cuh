// wavenet_lat.cuh -- the MODEL-SPECIALISED LOW-LATENCY WaveNet kernel for sm_90a: few streams, short calls.
//
// The reference's hosts call DSP::process() with ONE stream and 64-frame blocks (tools/benchmodel.cpp:116-133,
// NeuralAmpModelerPlugin): such a call is pure latency.  The precompiled kernel walks it with one frame per thread of a
// 128-thread CTA (half of them idle at 64 frames), ~22 layer steps each as long as one warp's whole instruction stream
// for a layer.
//
// This kernel is compiled per model by NVRTC like wavenet_spec.cuh (same generated header: namespace `spec`, weights as
// FFMA immediates) and cuts the step three ways:
//   * a layer's OUTPUT CHANNELS are split over 4 warp groups: thread (frame f, group g) computes channels
//     [g C/4, (g+1) C/4) of frame f -- a quarter of the layer's FMAs per thread.  Each group has its own instruction
//     stream (its own immediates): the four copies of the layer loop together are as large as one full copy.  What
//     needs all channels of a frame (the 1x1 after the activation, the head rechannel, the next array's rechannel)
//     goes through a shared-memory exchange of the frame's column: one extra barrier per layer;
//   * ALL history the call needs is requested at kernel start: for every (layer, tap) the window of ring columns
//     [t0 - off, t0 - off + min(off, n)) is copied global -> shared by cp.async.bulk (UBLKCP) completing on that layer's
//     own mbarrier, so the L2 round trips of all layers overlap each other and the first layers' arithmetic instead of
//     being paid once per layer;
//   * no shared-memory weights to load at kernel start (55 KB per call for the precompiled kernel).
// Same rings, same arithmetic order per output as wavenet_fused.cuh / wavenet_spec.cuh, so calls can be mixed.
//
// Geometry: one CTA per stream, FW frame warps (frames per call <= 32 FW), 4 or 8 channel groups: 128 FW / 256 FW threads.
#pragma once

#ifndef NAMB200_SPEC_HEADER_INCLUDED
#error "include the generated model header (namespace spec) before wavenet_lat.cuh"
#endif

#define NAMB200_SPEC_NO_KERNEL 1
#include "wavenet_spec.cuh" // helpers (activations, mbarrier / bulk-copy primitives, static_for); its kernel is compiled out

namespace namb200_lat
{
using namespace namb200_spec;

#ifndef NAMB200_LAT_GROUPS
#define NAMB200_LAT_GROUPS 4
#endif
// Channel groups.  Each group is its own instruction stream, and streaming straight-line code from L2 is what bounds this
// kernel: an SM fetches more bytes per cycle from more distinct code streams, so 8 groups of half-size streams finish
// sooner than 4.
constexpr int kGroups = NAMB200_LAT_GROUPS;
static_assert(kGroups == 4 || kGroups == 8, "4 or 8 channel groups");

struct LatParams
{
  float* state; // [batch][state_stride]
  long state_stride;
  const float* in; // [batch][in_stride] (may be mapped host memory)
  float* out;
  long in_stride, out_stride;
  int batch, n_frames; // n_frames <= 32 * FW
  u32 t_base;
  // completion doorbell (may be null): a word in mapped host memory that receives `seq` once every output of the call
  // is visible to the host -- the host spins on it instead of paying a stream synchronisation per 64-frame call
  unsigned* done_flag;
  unsigned seq;
};

// ---- shared-memory plan (float4 columns) ------------------------------------------------------------------------------
//   tile [Pmax][F]   the current layer's input columns of this call
//   xbuf [Pmax][F]   exchange: a frame's activations (and head sums) for the threads of the other channel groups
//   win  (layer, tap) windows, P_l planes x wn columns each, wn = min(off, F)
template <int F>
struct Plan
{
  __host__ __device__ static constexpr int pmax()
  {
    int p = 0;
    for (int a = 0; a < spec::NA; a++)
      p = spec::A[a].C / 4 > p ? spec::A[a].C / 4 : p;
    return p;
  }
  __host__ __device__ static constexpr int wn(int li, int k) // columns of the window of tap k of layer li
  {
    const int off = (spec::L[li].K - 1 - k) * spec::L[li].dil;
    return off < F ? off : F;
  }
  __host__ __device__ static constexpr int win_off(int li, int k) // float4 offset of that window inside the window area
  {
    int o = 0;
    for (int l = 0; l < spec::NL; l++)
      for (int kk = 0; kk < spec::L[l].K - 1; kk++)
      {
        if (l == li && kk == k)
          return o;
        o += (spec::layer_channels(l) / 4) * wn(l, kk);
      }
    return o;
  }
  __host__ __device__ static constexpr int win_total()
  {
    int o = 0;
    for (int l = 0; l < spec::NL; l++)
      for (int kk = 0; kk < spec::L[l].K - 1; kk++)
        o += (spec::layer_channels(l) / 4) * wn(l, kk);
    return o;
  }
  __host__ __device__ static constexpr int layer_bytes(int li) // what the layer's mbarrier waits for
  {
    int b = 0;
    for (int kk = 0; kk < spec::L[li].K - 1; kk++)
      b += (spec::layer_channels(li) / 4) * wn(li, kk) * 16;
    return b;
  }
  __host__ __device__ static constexpr int total_float4() { return 2 * pmax() * F + win_total(); }
};

struct Ctx
{
  float4* tile;
  float4* xbuf;
  float4* win;
  u64* bars; // one mbarrier per layer
  float* state;
  u32 tabs0;
  int n; // frames of this call
  int f; // this thread's frame
};

// a group's CO consecutive channels <-> a slice of a 4-channel plane column
template <int CO>
__device__ __forceinline__ void store_slice(float4* planes, const int F, const int g, const int f, const float (&v)[CO])
{
  if constexpr (CO == 4)
    planes[g * F + f] = make_float4(v[0], v[1], v[2], v[3]);
  else if constexpr (CO == 2)
    reinterpret_cast<float2*>(planes + (g >> 1) * F + f)[g & 1] = make_float2(v[0], v[1]);
  else
    reinterpret_cast<float*>(planes + (g >> 2) * F + f)[g & 3] = v[0];
}
template <int CO>
__device__ __forceinline__ void load_slice(const float4* planes, const int F, const int g, const int f, float (&v)[CO])
{
  if constexpr (CO == 4)
  {
    const float4 q = planes[g * F + f];
    v[0] = q.x, v[1] = q.y, v[2] = q.z, v[3] = q.w;
  }
  else if constexpr (CO == 2)
  {
    const float2 q = reinterpret_cast<const float2*>(planes + (g >> 1) * F + f)[g & 1];
    v[0] = q.x, v[1] = q.y;
  }
  else
    v[0] = reinterpret_cast<const float*>(planes + (g >> 2) * F + f)[g & 3];
}
// all C channels of frame f
template <int C>
__device__ __forceinline__ void load_column(const float4* planes, const int F, const int f, float (&v)[C])
{
#pragma unroll
  for (int pl = 0; pl < C / 4; pl++)
  {
    const float4 q = planes[pl * F + f];
    v[4 * pl] = q.x, v[4 * pl + 1] = q.y, v[4 * pl + 2] = q.z, v[4 * pl + 3] = q.w;
  }
}

// the layer's activation on a slice of channels [ch0, ch0 + CO) of the frame
template <int LI, int C, int CO>
__device__ __forceinline__ void activate_slice(float (&v)[CO], const int ch0)
{
  if constexpr (spec::L[LI].act == ACT_FASTTANH)
  {
#pragma unroll
    for (int q = 0; q + 1 < CO; q += 2)
      unpack2(fast_tanh2(pack2(v[q], v[q + 1])), v[q], v[q + 1]);
    if constexpr (CO % 2 == 1)
    {
      float lo, hi;
      unpack2(fast_tanh2(pack2(v[CO - 1], 0.0f)), lo, hi);
      v[CO - 1] = lo;
    }
  }
  else
  {
#pragma unroll
    for (int o = 0; o < CO; o++)
      v[o] = act_scalar<LI, C>(v[o], ch0 + o); // (PReLU: per-channel slopes)
  }
}

// this group's slice of the ring column of frame f (plain stores: nobody waits for them; RingBuffer::Write semantics)
template <int C, int CO, int LI>
__device__ __forceinline__ void ring_store_slice(const Ctx& c, const int g, const float (&v)[CO])
{
  constexpr spec::Layer Ld = spec::L[LI];
  constexpr int R = Ld.ring_mask + 1;
  constexpr int L = (Ld.K - 1) * Ld.dil;
  // only the call's last `look-back` columns: the ring may have exactly that many slots, older columns would alias them
  if (c.f >= c.n || c.f < c.n - L)
    return;
  const u32 col = (c.tabs0 + (u32)c.f) & (u32)Ld.ring_mask;
  float* ring = c.state + Ld.ring_off;
  const int ch0 = g * CO; // first channel of the slice
  float* dst = ring + ((size_t)(ch0 >> 2) * R + col) * 4 + (ch0 & 3);
  if constexpr (CO == 4)
    __stcg(reinterpret_cast<float4*>(dst), make_float4(v[0], v[1], v[2], v[3]));
  else if constexpr (CO == 2)
    __stcg(reinterpret_cast<float2*>(dst), make_float2(v[0], v[1]));
  else
    __stcg(dst, v[0]);
}

// Every history window of the call, requested at kernel start.  Warp w takes the layers w, w + NW, ..: a bulk copy is issued
// through uniform registers, one at a time per warp (~40 cycles each), and a1_standard has 160 of them -- spread over the
// CTA's warps they cost a fraction of what one warp issuing them all would.
template <int F, int NWARPS>
__device__ __forceinline__ void request_all_history(const Ctx& c, const int warp, const int lane)
{
  static_for<0, spec::NL>([&](auto li_c) {
    constexpr int LI = decltype(li_c)::value;
    if (warp != LI % NWARPS) // (warp-uniform)
      return;
    constexpr spec::Layer Ld = spec::L[LI];
    constexpr int P = spec::layer_channels(LI) / 4, R = Ld.ring_mask + 1;
    constexpr int NW = Ld.K - 1;
    constexpr int bytes = Plan<F>::layer_bytes(LI); // (every index below is a constant expression: host-side tables)
    if (lane == 0)
      mbar_expect_tx(c.bars + LI, (u32)bytes);
    __syncwarp();
    const float4* ring = reinterpret_cast<const float4*>(c.state + Ld.ring_off);
    static_for<0, NW>([&](auto k_c) {
      constexpr int k = decltype(k_c)::value;
      constexpr int off = (Ld.K - 1 - k) * Ld.dil;
      constexpr int wn = Plan<F>::wn(LI, k);
      constexpr int woff = Plan<F>::win_off(LI, k);
      if (lane < P)
      {
        float4* dst = c.win + woff + lane * wn;
        const int start = (int)((c.tabs0 - (u32)off) & (u32)Ld.ring_mask);
        const int n1 = min(wn, R - start);
        bulk_g2s(dst, ring + lane * R + start, (u32)n1 * 16u, c.bars + LI);
        if (n1 < wn)
          bulk_g2s(dst + n1, ring + lane * R, (u32)(wn - n1) * 16u, c.bars + LI);
      }
    });
  });
}

// One layer array for thread (frame f, channel group G): channels [G CO, (G+1) CO), CO = C / 4.
//   hin[CIN]: ALL input channels of the frame; head[CO], headout[...]: this group's slices
template <int AI, int G, int F, int NTH>
__device__ __forceinline__ void array_forward_lat(Ctx& c, const float (&hin)[spec::A[AI].CIN], const float cond,
                                                  float (&head)[spec::A[AI].C / kGroups],
                                                  float (&hout_all)[spec::A[AI].C], float (&headout_all)[spec::A[AI].HOUT])
{
  constexpr spec::Array A = spec::A[AI];
  constexpr int C = A.C, CIN = A.CIN, HOUT = A.HOUT, P = C / 4, CO = C / kGroups;
  static_assert(A.head_kernel == 1, "convolutional heads are served by the generic fused kernel");
  static_assert(C % kGroups == 0, "channels are padded to 4 / 8 / 16");
  const int f = c.f;

  // ---- rechannel (Conv1x1, no bias; model.cpp:492): this group's channels of the layer-0 input
  float h[CO];
#pragma unroll
  for (int o = 0; o < CO; o++)
    h[o] = 0.0f;
#pragma unroll
  for (int i = 0; i < CIN; i++)
#pragma unroll
    for (int o = 0; o < CO; o++)
      h[o] = fmaf(spec::w(A.rech_off + i * C + G * CO + o), hin[i], h[o]);
  store_slice<CO>(c.tile, F, G, f, h);

  static_for<0, A.n_layers>([&](auto li_c) {
    constexpr int LI = A.layer0 + decltype(li_c)::value;
    constexpr bool last = (decltype(li_c)::value + 1 == A.n_layers);
    constexpr spec::Layer Ld = spec::L[LI];
    constexpr int K = Ld.K, dil = Ld.dil;
    constexpr int w_conv = Ld.w_off, w_bias = w_conv + K * C * C, w_mix = w_bias + C, w_p = w_mix + C, w_pb = w_p + C * C;

    __syncthreads(); // B0: the layer input is complete in the tile (and xbuf reads of the previous layer are done)
    mbar_wait(c.bars + LI, 0u); // this layer's history windows have landed (each barrier is used once per launch)

    // my slice of the layer input goes to the ring; it is also the residual
    float own[CO];
    load_slice<CO>(c.tile, F, G, f, own);
    ring_store_slice<C, CO, LI>(c, G, own);

    // ---- z = b + M c + sum_k W_k h[t - (K-1-k) d];  a = act(z);  head += a   (this group's channels)
    float acc[CO];
#pragma unroll
    for (int o = 0; o < CO; o++)
      acc[o] = fmaf(spec::w(w_mix + G * CO + o), cond, spec::w(w_bias + G * CO + o));
    static_for<0, K>([&](auto k_c) {
      constexpr int k = decltype(k_c)::value;
      constexpr int off = (K - 1 - k) * dil;
      constexpr int wn = off < F ? off : F;
      constexpr int woff = (k < K - 1) ? Plan<F>::win_off(LI, k < K - 1 ? k : 0) : 0;
      // frames before `off` read the history window, the others the tile (one address select, no divergence)
      const bool hist = (off > 0) && (f < off);
      const float4* src = hist ? c.win + woff + f : c.tile + (f - off);
      const int stride = hist ? wn : F;
#pragma unroll
      for (int pl = 0; pl < P; pl++)
      {
        const float4 q = src[pl * stride];
        const float x[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int o = 0; o < CO; o++)
            acc[o] = fmaf(spec::w(w_conv + (k * C + 4 * pl + i) * C + G * CO + o), x[i], acc[o]);
      }
    });
    activate_slice<LI, C, CO>(acc, G * CO);
#pragma unroll
    for (int o = 0; o < CO; o++)
      head[o] += acc[o]; // model.cpp:530
    store_slice<CO>(c.xbuf, F, G, f, acc);
    __syncthreads(); // B_a: every group's activations of the frame are in xbuf; every tap read of the tile is done

    // ---- h_{l+1} = h_l + p + P a  (model.cpp:243,376): needs all C activations of the frame
    float a[C];
    load_column<C>(c.xbuf, F, f, a);
    float hn[CO];
#pragma unroll
    for (int o = 0; o < CO; o++)
      hn[o] = own[o] + spec::w(w_pb + G * CO + o);
#pragma unroll
    for (int i = 0; i < C; i++)
#pragma unroll
      for (int o = 0; o < CO; o++)
        hn[o] = fmaf(spec::w(w_p + i * C + G * CO + o), a[i], hn[o]);
    store_slice<CO>(c.tile, F, G, f, hn); // (the last layer's output: read back below as the array output)
  });

  // ---- array outputs need all channels of the frame: the last layer's output and the head accumulator
  __syncthreads();
  load_column<C>(c.tile, F, f, hout_all);
  store_slice<CO>(c.xbuf, F, G, f, head);
  __syncthreads();
  float hd[C];
  load_column<C>(c.xbuf, F, f, hd);
  // head rechannel (kernel size 1; model.cpp:548): every thread computes all HOUT outputs (HOUT <= 16: a few FMAs) so
  // that no further exchange is needed
#pragma unroll
  for (int ho = 0; ho < HOUT; ho++)
    headout_all[ho] = 0.0f;
#pragma unroll
  for (int i = 0; i < C; i++)
#pragma unroll
    for (int ho = 0; ho < HOUT; ho++)
      headout_all[ho] = fmaf(spec::w(A.head_off + i * HOUT + ho), hd[i], headout_all[ho]);
#pragma unroll
  for (int ho = 0; ho < HOUT; ho++)
    headout_all[ho] += spec::w(A.head_off + C * HOUT + ho);
}

template <int G, int F, int NTH>
__device__ __forceinline__ void network_lat(Ctx& c, const LatParams& p, const float x, float* yout, const int t_off)
{
  const float hin0[1] = {x};
  constexpr int C0 = spec::A[0].C;
  float head0[C0 / kGroups], hout0[C0], ho0[spec::A[0].HOUT];
#pragma unroll
  for (int o = 0; o < C0 / kGroups; o++)
    head0[o] = 0.0f; // model.cpp:469
  float y;
  array_forward_lat<0, G, F, NTH>(c, hin0, x, head0, hout0, ho0);
  if constexpr (spec::NA == 1)
    y = ho0[0];
  else
  {
    // second array: layer input = the previous array's layer output, head accumulator starts from the previous array's
    // head output (model.cpp:846-848, :473-486): this group's slice of it
    constexpr int AI1 = spec::NA - 1;
    constexpr int C1 = spec::A[AI1].C, CO1 = C1 / kGroups;
    float head1[CO1], hout1[C1], ho1[spec::A[AI1].HOUT];
#pragma unroll
    for (int o = 0; o < CO1; o++)
      head1[o] = ho0[G * CO1 + o];
    __syncthreads(); // the tile / xbuf columns read above are rewritten by the next array's rechannel
    array_forward_lat<AI1, G, F, NTH>(c, hout0, x, head1, hout1, ho1);
    y = ho1[0];
  }
  if (G == 0 && c.f < c.n)
    yout[t_off + c.f] = spec::head_scale * y; // model.cpp:888-897
}

template <int FW>
__device__ __forceinline__ void wavenet_lat_body(const LatParams& p)
{
  constexpr int F = 32 * FW, NTH = kGroups * F;
  static_assert(spec::NA == 1 || spec::NA == 2, "one or two layer arrays");
  extern __shared__ float4 lat_smem[];
  __shared__ u64 bars[spec::NL];
  const int tid = threadIdx.x;
  const int stream = blockIdx.x;
  Ctx c;
  c.tile = lat_smem;
  c.xbuf = lat_smem + Plan<F>::pmax() * F;
  c.win = lat_smem + 2 * Plan<F>::pmax() * F;
  c.bars = bars;
  c.state = p.state + (size_t)stream * p.state_stride;
  c.tabs0 = p.t_base;
  c.n = p.n_frames;
  c.f = tid & (F - 1);
  const int g = tid / F; // warp-uniform: F is a multiple of 32
  if (tid < spec::NL)
    mbar_init(bars + tid, 1);
  if (tid == 0)
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  request_all_history<F, NTH / 32>(c, tid >> 5, tid & 31);
  const float x = (c.f < c.n) ? p.in[(size_t)stream * p.in_stride + c.f] : 0.0f;
  float* yout = p.out + (size_t)stream * p.out_stride;
  // each channel group runs its own copy of the network: its weights are its own immediates
  static_for<0, kGroups>([&](auto g_c) {
    constexpr int G = decltype(g_c)::value;
    if (g == G)
      network_lat<G, F, NTH>(c, p, x, yout, 0);
  });
  if (p.done_flag != nullptr)
  {
    // barrier, then ONE system-scope fence by the signalling thread (fences are cumulative: it orders every output store the
    // barrier made it observe before the doorbell -- the grid-sync idiom); a fence by every thread before the barrier as well
    // only puts a second system-scope fence on the critical path
    __syncthreads();
    if (tid == 0 && blockIdx.x == 0)
    {
      __threadfence_system();
      *reinterpret_cast<volatile unsigned*>(p.done_flag) = p.seq;
    }
  }
}

} // namespace namb200_lat

#ifndef NAMB200_LAT_FW
#define NAMB200_LAT_FW 2
#endif

extern "C" __global__ void __launch_bounds__(32 * NAMB200_LAT_GROUPS * NAMB200_LAT_FW, 1)
  wavenet_lat_kernel(const __grid_constant__ namb200_lat::LatParams p)
{
  namb200_lat::wavenet_lat_body<NAMB200_LAT_FW>(p);
}
