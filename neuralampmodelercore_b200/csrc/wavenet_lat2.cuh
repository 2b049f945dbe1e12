// wavenet_lat2.cuh -- the low-latency WaveNet kernel, precompiled: few streams, short calls (the plugin protocol).
//
// Reference path: the same as wavenet_fused.cuh (NAM/wavenet/model.cpp:822-910, :463-549, :183-393; conv1d.cpp:666-683;
// ring_buffer.cpp:7-109; dsp.cpp:436-836; activations.h:59-133).
//
// What limits its two predecessors on ONE stream x 64 frames of wavenet_a1_standard.nam:
//   * the 128 x 1 geometry of wavenet_fused.cuh: ~22 layer steps, each one warp's whole
//     instruction stream for a layer, half the CTA idle at 64 frames, the L2 round trip of the ring columns paid per layer;
//   * the model-specialised wavenet_lat.cuh (weights as FFMA immediates, output channels split over four warp groups, all
//     history requested at kernel start): a few hundred KB of straight-line code executed exactly once per call is an
//     instruction-fetch stream.
// This kernel keeps the two things that worked (channel groups over warps; every history window of the call requested at
// kernel start by cp.async.bulk, one mbarrier per layer) and moves the weights back to DATA: ONE bulk copy brings the
// whole 55 KB blob into shared memory per call (the data path moves it in ~0.6 us; the instruction path needed ~10), and
// the layer loop is rolled: a few KB of code that stays in the instruction cache.  A group's four output-channel weights
// of an input channel are one warp-uniform LDS.128.
//
// Geometry: one CTA per stream, FW frame warps x 4 channel groups = 128 FW threads; calls of up to 32 FW frames.
#pragma once

#include "wavenet_fused.cuh"

namespace namb200
{

constexpr int kLatGroups = 4;

// ---- mbarrier / bulk-copy primitives (cf. wavenet_spec.cuh) --------------------------------------------------------------
__device__ __forceinline__ uint32_t lat_smem_addr(const void* p)
{
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void lat_mbar_init(uint64_t* bar, int count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(lat_smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void lat_mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(lat_smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void lat_mbar_wait(uint64_t* bar, uint32_t parity)
{
  asm volatile(
    "{\n"
    ".reg .pred p;\n"
    "WAIT_%=:\n"
    "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
    "@p bra DONE_%=;\n"
    "bra WAIT_%=;\n"
    "DONE_%=:\n"
    "}\n" ::"r"(lat_smem_addr(bar)),
    "r"(parity)
    : "memory");
}
__device__ __forceinline__ void lat_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                 lat_smem_addr(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(lat_smem_addr(bar))
               : "memory");
}

// shared-memory plan (float4 units): weights | tile [Pmax][F] | xbuf [Pmax][F] | windows
__host__ __device__ inline int lat2_window_cols(int off, int F)
{
  return off < F ? off : F;
}

struct Lat2Ctx
{
  const float* w; // the weight blob in shared memory
  float4* tile;
  float4* xbuf;
  float4* win;
  const int* woff; // [layer]: float4 offset of the layer's first window inside `win` (shared memory)
  uint64_t* bars; // [layer]
  float* state;
  uint32_t tabs0;
  int n, f, g;
};

template <int CO>
__device__ __forceinline__ void lat2_store_slice(float4* planes, const int F, const int g, const int f, const float (&v)[CO])
{
  if constexpr (CO == 4)
    planes[g * F + f] = make_float4(v[0], v[1], v[2], v[3]);
  else if constexpr (CO == 2)
    reinterpret_cast<float2*>(planes + (g >> 1) * F + f)[g & 1] = make_float2(v[0], v[1]);
  else
    reinterpret_cast<float*>(planes + f)[g] = v[0];
}
template <int CO>
__device__ __forceinline__ void lat2_load_slice(const float4* planes, const int F, const int g, const int f, float (&v)[CO])
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
    v[0] = reinterpret_cast<const float*>(planes + f)[g];
}
// CO consecutive weights (a group's output channels of one input channel): one warp-uniform load
template <int CO>
__device__ __forceinline__ void lat2_load_w(const float* p, float (&v)[CO])
{
  if constexpr (CO == 4)
  {
    const float4 q = *reinterpret_cast<const float4*>(p);
    v[0] = q.x, v[1] = q.y, v[2] = q.z, v[3] = q.w;
  }
  else if constexpr (CO == 2)
  {
    const float2 q = *reinterpret_cast<const float2*>(p);
    v[0] = q.x, v[1] = q.y;
  }
  else
    v[0] = *p;
}

// One layer array for thread (frame f, channel group g): channels [g CO, (g+1) CO), CO = C / 4.
template <int CIN, int C, int HOUT, int F>
__device__ __forceinline__ void lat2_array(const WaveNetKernelParams& p, const ArrayDesc& A, const Lat2Ctx& c,
                                           const float (&hin)[CIN], const float cond, float (&head)[C / kLatGroups],
                                           float (&hout_all)[C], float (&headout_all)[HOUT])
{
  constexpr int P = C / 4, CO = C / kLatGroups;
  const int f = c.f, g = c.g;
  {
    float h[CO];
#pragma unroll
    for (int o = 0; o < CO; o++)
      h[o] = 0.0f;
#pragma unroll
    for (int i = 0; i < CIN; i++)
    {
      float wv[CO];
      lat2_load_w<CO>(c.w + A.rech_off + i * C + g * CO, wv);
#pragma unroll
      for (int o = 0; o < CO; o++)
        h[o] = fmaf(wv[o], hin[i], h[o]);
    }
    lat2_store_slice<CO>(c.tile, F, g, f, h);
  }

#pragma unroll 1
  for (int li = 0; li < A.n_layers; li++)
  {
    const int LI = A.layer0 + li;
    const LayerDesc& Ld = p.layers[LI];
    const int K = Ld.kernel, dil = Ld.dilation, L = Ld.lookback, R = Ld.ring_mask + 1;
    const float* __restrict__ w = c.w + Ld.w_off;
    const float* __restrict__ w_bias = w + K * C * C;
    const float* __restrict__ w_mix = w_bias + C;
    const float* __restrict__ w_p = w_mix + C;
    const float* __restrict__ w_pb = w_p + C * C;
    const float* __restrict__ w_slopes = w_pb + C;

    __syncthreads(); // B0: the layer input is complete in the tile
    lat_mbar_wait(c.bars + LI, 0u); // this layer's history windows have landed

    float own[CO];
    lat2_load_slice<CO>(c.tile, F, g, f, own);
    if (f < c.n && f >= c.n - L) // RingBuffer::Write: the call's last `look-back` columns
    {
      const uint32_t col = (c.tabs0 + (uint32_t)f) & (uint32_t)Ld.ring_mask;
      const int ch0 = g * CO;
      float* dst = c.state + Ld.ring_off + ((size_t)(ch0 >> 2) * R + col) * 4 + (ch0 & 3);
      if constexpr (CO == 4)
        __stcg(reinterpret_cast<float4*>(dst), make_float4(own[0], own[1], own[2], own[3]));
      else if constexpr (CO == 2)
        __stcg(reinterpret_cast<float2*>(dst), make_float2(own[0], own[1]));
      else
        __stcg(dst, own[0]);
    }

    float acc[CO];
    {
      float b[CO], mw[CO];
      lat2_load_w<CO>(w_bias + g * CO, b);
      lat2_load_w<CO>(w_mix + g * CO, mw);
#pragma unroll
      for (int o = 0; o < CO; o++)
        acc[o] = fmaf(mw[o], cond, b[o]);
    }
    int wbase = c.woff[LI];
    auto tap = [&](const int k) {
      const int off = (K - 1 - k) * dil;
      const int wn = lat2_window_cols(off, F);
      const bool hist = (off > 0) && (f < off);
      const float4* src = hist ? c.win + wbase + f : c.tile + (f - off);
      const int stride = hist ? wn : F;
      const float* __restrict__ wk = w + (size_t)k * C * C + g * CO;
#pragma unroll
      for (int pl = 0; pl < P; pl++)
      {
        const float4 q = src[pl * stride];
        const float x[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int i = 0; i < 4; i++)
        {
          float wv[CO];
          lat2_load_w<CO>(wk + (4 * pl + i) * C, wv);
#pragma unroll
          for (int o = 0; o < CO; o++)
            acc[o] = fmaf(wv[o], x[i], acc[o]);
        }
      }
      if (off > 0)
        wbase += P * wn;
    };
    if (K == 3) // the kernel size of the classic family: unrolled, so the loads of the three taps overlap
    {
      tap(0);
      tap(1);
      tap(2);
    }
    else
    {
#pragma unroll 1
      for (int k = 0; k < K; k++)
        tap(k);
    }
    // activation on this group's channels (PReLU: the group's slopes)
    if (Ld.act == KACT_FASTTANH)
    {
      if constexpr (CO >= 2)
      {
#pragma unroll
        for (int q = 0; q < CO / 2; q++)
          unpack2(tc_fast_tanh2(pack2(acc[2 * q], acc[2 * q + 1])), acc[2 * q], acc[2 * q + 1]);
      }
      else
        acc[0] = act_fast_tanh(acc[0]);
    }
    else
      apply_activation<CO>(acc, Ld, w_slopes + g * CO);
#pragma unroll
    for (int o = 0; o < CO; o++)
      head[o] += acc[o]; // model.cpp:530
    lat2_store_slice<CO>(c.xbuf, F, g, f, acc);
    __syncthreads(); // B_a: the frame's activations of all groups are in xbuf; every tap read of the tile is done

    float hn[CO];
    {
      float pb[CO];
      lat2_load_w<CO>(w_pb + g * CO, pb);
#pragma unroll
      for (int o = 0; o < CO; o++)
        hn[o] = own[o] + pb[o];
    }
#pragma unroll
    for (int pl = 0; pl < P; pl++)
    {
      const float4 q = c.xbuf[pl * F + f];
      const float a[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int i = 0; i < 4; i++)
      {
        float wv[CO];
        lat2_load_w<CO>(w_p + (4 * pl + i) * C + g * CO, wv);
#pragma unroll
        for (int o = 0; o < CO; o++)
          hn[o] = fmaf(wv[o], a[i], hn[o]);
      }
    }
    lat2_store_slice<CO>(c.tile, F, g, f, hn);
  }

  // array outputs need all channels of the frame: the last layer's output and the head accumulator
  __syncthreads();
#pragma unroll
  for (int pl = 0; pl < P; pl++)
  {
    const float4 q = c.tile[pl * F + f];
    hout_all[4 * pl] = q.x, hout_all[4 * pl + 1] = q.y, hout_all[4 * pl + 2] = q.z, hout_all[4 * pl + 3] = q.w;
  }
  lat2_store_slice<CO>(c.xbuf, F, g, f, head);
  __syncthreads();
  const float* __restrict__ wh = c.w + A.head_off;
#pragma unroll
  for (int ho = 0; ho < HOUT; ho++)
    headout_all[ho] = 0.0f;
#pragma unroll
  for (int pl = 0; pl < P; pl++)
  {
    const float4 q = c.xbuf[pl * F + f];
    const float hd[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int ho = 0; ho < HOUT; ho++)
        headout_all[ho] = fmaf(wh[(4 * pl + i) * HOUT + ho], hd[i], headout_all[ho]);
  }
#pragma unroll
  for (int ho = 0; ho < HOUT; ho++)
    headout_all[ho] += wh[C * HOUT + ho]; // (zero when the head has no bias)
}

// One CTA per stream; C1 == 0: single layer array.  The completion doorbell (p.done_flag, may be null) is rung once the
// outputs are visible to the host.
// TBL: the call carries a slot table (its own instantiation: a call without one runs the table-free code).
template <int C0, int C1, int FW, bool TBL = false>
__global__ void __launch_bounds__(128 * FW, 1) wavenet_lat2_kernel(const __grid_constant__ WaveNetKernelParams p)
{
  constexpr int F = 32 * FW, NTH = kLatGroups * F, NWARPS = NTH / 32;
  constexpr int PMAX = (C0 > C1 ? C0 : C1) / 4;
  extern __shared__ float4 lat2_smem[];
  __shared__ uint64_t bars[kMaxLayers + 1]; // [layer] windows; [kMaxLayers] the weight blob
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_layers = p.arrays[0].n_layers + (C1 != 0 ? p.arrays[1].n_layers : 0);
  const int wf4 = (p.n_weight_floats + 3) / 4;
  float4* const tile = lat2_smem + wf4;
  float4* const xbuf = tile + PMAX * F;
  float4* const win = xbuf + PMAX * F;
  const int stream = blockIdx.x; // position in the call (input / output row)
  float* const state = p.state + (size_t)(TBL ? p.slots[stream].stream : stream) * p.state_stride;
  const uint32_t clock = TBL ? p.slots[stream].clock : p.t_base; // where this stream's history ends
  const int model = TBL ? p.slots[stream].model : 0; // a bank's stream brings its own model's blob and output scale

  // window table: float4 offset of each layer's first window (prefix sums, thread li computes entry li) -- it lives
  // behind the windows; total window size is bounded by the host (lat2_smem_bytes)
  int win_total = 0;
  {
    // every thread walks the (short) layer list once: the prefix it needs is its own layer's for li = tid
    int acc_cols = 0;
    for (int a = 0; a < (C1 != 0 ? 2 : 1); a++)
    {
      const int Pa = (a == 0 ? C0 : C1) / 4;
      for (int i = 0; i < p.arrays[a].n_layers; i++)
      {
        const LayerDesc& Ld = p.layers[p.arrays[a].layer0 + i];
        for (int k = 0; k + 1 < Ld.kernel; k++)
          acc_cols += Pa * lat2_window_cols((Ld.kernel - 1 - k) * Ld.dilation, F);
      }
    }
    win_total = acc_cols;
  }
  int* const woff = reinterpret_cast<int*>(win + win_total);
  if (tid < n_layers)
  {
    int acc_cols = 0, idx = 0;
    for (int a = 0; a < (C1 != 0 ? 2 : 1); a++)
    {
      const int Pa = (a == 0 ? C0 : C1) / 4;
      for (int i = 0; i < p.arrays[a].n_layers; i++, idx++)
      {
        const LayerDesc& Ld = p.layers[p.arrays[a].layer0 + i];
        if (p.arrays[a].layer0 + i == tid)
          woff[tid] = acc_cols;
        for (int k = 0; k + 1 < Ld.kernel; k++)
          acc_cols += Pa * lat2_window_cols((Ld.kernel - 1 - k) * Ld.dilation, F);
      }
    }
    lat_mbar_init(bars + tid, 1);
  }
  if (tid == 0)
  {
    lat_mbar_init(bars + kMaxLayers, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // ---- requests: the weight blob (one copy) and every history window of the call (warp w: layers w, w + NWARPS, ..)
  if (tid == 0)
  {
    lat_mbar_expect_tx(bars + kMaxLayers, (uint32_t)wf4 * 16u);
    lat_bulk_g2s(lat2_smem, TBL ? p.weights + (size_t)model * p.weight_stride : p.weights, (uint32_t)wf4 * 16u, bars + kMaxLayers);
  }
  for (int a = 0; a < (C1 != 0 ? 2 : 1); a++)
  {
    const int Pa = (a == 0 ? C0 : C1) / 4;
    for (int i = 0; i < p.arrays[a].n_layers; i++)
    {
      const int LI = p.arrays[a].layer0 + i;
      if ((LI % NWARPS) != warp)
        continue;
      const LayerDesc& Ld = p.layers[LI];
      const int R = Ld.ring_mask + 1;
      int bytes = 0;
      for (int k = 0; k + 1 < Ld.kernel; k++)
        bytes += Pa * lat2_window_cols((Ld.kernel - 1 - k) * Ld.dilation, F) * 16;
      if (lane == 0)
        lat_mbar_expect_tx(bars + LI, (uint32_t)bytes);
      __syncwarp();
      const float4* ring = reinterpret_cast<const float4*>(state + Ld.ring_off);
      int base = woff[LI];
      for (int k = 0; k + 1 < Ld.kernel; k++)
      {
        const int off = (Ld.kernel - 1 - k) * Ld.dilation;
        const int wn = lat2_window_cols(off, F);
        if (lane < Pa)
        {
          float4* dst = win + base + lane * wn;
          const int start = (int)((clock - (uint32_t)off) & (uint32_t)Ld.ring_mask);
          const int n1 = min(wn, R - start);
          lat_bulk_g2s(dst, ring + lane * R + start, (uint32_t)n1 * 16u, bars + LI);
          if (n1 < wn)
            lat_bulk_g2s(dst + n1, ring + lane * R, (uint32_t)(wn - n1) * 16u, bars + LI);
        }
        base += Pa * wn;
      }
    }
  }

  Lat2Ctx c;
  c.w = reinterpret_cast<const float*>(lat2_smem);
  c.tile = tile;
  c.xbuf = xbuf;
  c.win = win;
  c.woff = woff;
  c.bars = bars;
  c.state = state;
  c.tabs0 = clock;
  c.n = TBL ? p.slots[stream].frames : p.n_frames; // (one stream per CTA: its own count)
  c.f = tid & (F - 1);
  c.g = tid / F;
  const float xv = (c.f < c.n) ? p.in[(size_t)stream * p.in_stride + c.f] : 0.0f;
  lat_mbar_wait(bars + kMaxLayers, 0u); // the weights are in shared memory

  const float hin0[1] = {xv};
  float y;
  if constexpr (C1 == 0)
  {
    float head0[C0 / kLatGroups], hout0[C0], ho0[1];
#pragma unroll
    for (int o = 0; o < C0 / kLatGroups; o++)
      head0[o] = 0.0f;
    lat2_array<1, C0, 1, F>(p, p.arrays[0], c, hin0, xv, head0, hout0, ho0);
    y = ho0[0];
  }
  else
  {
    float head0[C0 / kLatGroups], hout0[C0], ho0[C1];
#pragma unroll
    for (int o = 0; o < C0 / kLatGroups; o++)
      head0[o] = 0.0f;
    lat2_array<1, C0, C1, F>(p, p.arrays[0], c, hin0, xv, head0, hout0, ho0);
    constexpr int CO1 = C1 / kLatGroups;
    float head1[CO1], hout1[C1], ho1[1];
#pragma unroll
    for (int o = 0; o < CO1; o++)
    {
      head1[o] = 0.0f;
#pragma unroll
      for (int gg = 0; gg < kLatGroups; gg++) // (a select chain: a register array cannot be indexed by the run-time group)
        if (c.g == gg)
          head1[o] = ho0[gg * CO1 + o]; // model.cpp:846-848, :473-486
    }
    __syncthreads();
    lat2_array<C0, C1, 1, F>(p, p.arrays[1], c, hout0, xv, head1, hout1, ho1);
    y = ho1[0];
  }
  if (c.g == 0 && c.f < c.n)
    p.out[(size_t)stream * p.out_stride + c.f] = (TBL && p.head_scales ? p.head_scales[model] : p.head_scale) * y; // model.cpp:888-897
  if (p.done_flag != nullptr)
  {
    // barrier, then ONE system-scope fence by the signalling thread (fences are cumulative: it orders every output store the
    // barrier made it observe before the doorbell -- the grid-sync idiom); a fence by every thread before the barrier as well
    // only puts a second system-scope fence on the critical path
    __syncthreads();
    if (tid == 0 && blockIdx.x == 0)
    {
      __threadfence_system();
      *reinterpret_cast<volatile unsigned*>(p.done_flag) = p.done_seq;
    }
  }
}

} // namespace namb200
