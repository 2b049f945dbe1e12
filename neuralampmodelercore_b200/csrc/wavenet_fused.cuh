// wavenet_fused.cuh -- the fused WaveNet layer-array kernel for sm_90a.
//
// What it replaces (reference file:line, all under NAM/):
//   wavenet/model.cpp:822-910   WaveNet::process            (whole kernel)
//   wavenet/model.cpp:463-549   LayerArray::Process{,Inner} (array_forward)
//   wavenet/model.cpp:183-393   Layer::Process, non-gated / no-FiLM / no-head1x1 path
//   conv1d.cpp:163-183,666-683,769-774  Conv1D::Process     (tap loop, history)
//   ring_buffer.cpp:7-109       RingBuffer                  (per-stream device rings)
//   dsp.cpp:436-836             Conv1x1::process_           (rechannel / mixin / layer1x1 / head)
//   activations.h:59-133        scalar activations
//
// Reframing (not a port): the reference walks ONE stream, layer by layer, over a 64-frame
// block with ~65 small GEMM calls.  Here one CTA owns one stream at a time and a tile of
// T = S*NT consecutive frames; THREAD t owns time steps {t, t+NT, ...} for the whole depth of
// the network.  With that mapping everything in a layer except the dilated taps is
// thread-local -- conv accumulate, +mixin, activation, head accumulate, 1x1, residual -- so
// activations never leave registers, and the only cross-thread traffic is "my column of the
// layer input" -> shared memory -> "columns t-d, t-2d of other threads".  Taps that reach
// behind the tile come from the stream's history rings in global memory; a persistent CTA
// keeps one stream's rings (196 KB for the standard model) L2-resident while it works
// through that stream's frames.
//
// Data layout: activations everywhere are "planes of 4 channels": [C/4][time][4 floats], so a
// thread's 16-byte vector load of (time, 4 channels) is contiguous across the warp's 32
// consecutive time steps (conflict-free LDS.128 / fully coalesced LDG.128), at ANY tap
// offset.  Weights live in shared memory as [in][out] rows so one warp-uniform LDS.128 yields 4
// output-channel weights, consumed two output channels at a time (a register pair, input sample
// broadcast; two scalar FFMAs on sm_90).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "wavenet_desc.h"

// unroll factor of the per-tap plane loop (4 input channels per plane): full unroll removes the
// loop-carried accumulator copies ptxas otherwise inserts at the back-edge
#ifndef NAMB200_PL_UNROLL
#define NAMB200_PL_UNROLL 4
#endif

namespace namb200
{
constexpr int kPlUnroll = NAMB200_PL_UNROLL;

// ---- activations ---------------------------------------------------------------------------
// Quotients use MUFU.RCP (<= 1 ulp) times the numerator instead of an IEEE division: every denominator below
// is >= 1, so neither the division slow path nor __fdividef's denormal-range rescaling (3 extra instructions
// per element) is needed.  Measured against the oracle in tests/test_parity_gpu.py.
__device__ __forceinline__ float rcp_approx(float x)
{
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// fast_tanh: the reference's rational approximation (activations.h:91-98); denominator >= 2.445.
__device__ __forceinline__ float act_fast_tanh(float x)
{
  const float ax = fabsf(x);
  const float x2 = x * x;
  const float num = x * (2.45550750702956f + 2.45550750702956f * ax + (0.893229853513558f + 0.821226666969744f * ax) * x2);
  const float den = 2.44506634652299f + (2.44506634652299f + x2) * fabsf(x + 0.814642734961073f * x * ax);
  return num * rcp_approx(den);
}

// sigmoid(x) = 1/(1+expf(-x)) (activations.h:64-67)
__device__ __forceinline__ float act_sigmoid(float x)
{
  return rcp_approx(1.0f + expf(-x));
}

template <int N>
__device__ __forceinline__ void apply_activation(float (&v)[N], const LayerDesc& L, const float* __restrict__ slopes)
{
  switch (L.act)
  {
    case KACT_TANH:
#pragma unroll
      for (int i = 0; i < N; i++)
        v[i] = tanhf(v[i]);
      break;
    case KACT_FASTTANH:
#pragma unroll
      for (int i = 0; i < N; i++)
        v[i] = act_fast_tanh(v[i]);
      break;
    case KACT_HARDTANH:
#pragma unroll
      for (int i = 0; i < N; i++)
        v[i] = fminf(fmaxf(v[i], -1.0f), 1.0f);
      break;
    case KACT_RELU:
#pragma unroll
      for (int i = 0; i < N; i++)
        v[i] = v[i] > 0.0f ? v[i] : 0.0f;
      break;
    case KACT_LEAKYRELU:
#pragma unroll
      for (int i = 0; i < N; i++)
        v[i] = v[i] > 0.0f ? v[i] : L.ap0 * v[i];
      break;
    case KACT_PRELU:
#pragma unroll
      for (int i = 0; i < N; i++)
        v[i] = v[i] > 0.0f ? v[i] : slopes[i] * v[i];
      break;
    case KACT_SIGMOID:
#pragma unroll
      for (int i = 0; i < N; i++)
        v[i] = act_sigmoid(v[i]);
      break;
    case KACT_SILU:
#pragma unroll
      for (int i = 0; i < N; i++)
        v[i] = v[i] * act_sigmoid(v[i]);
      break;
    case KACT_HARDSWISH:
#pragma unroll
      for (int i = 0; i < N; i++)
      {
        const float t = v[i] + 3.0f;
        const float cl = t < 0.0f ? 0.0f : (t > 6.0f ? 6.0f : t);
        v[i] = v[i] * cl * (1.0f / 6.0f);
      }
      break;
    case KACT_LEAKYHARDTANH:
#pragma unroll
      for (int i = 0; i < N; i++)
      {
        const float x = v[i];
        v[i] = x < L.ap0 ? (x - L.ap0) * L.ap2 + L.ap0 : (x > L.ap1 ? (x - L.ap1) * L.ap3 + L.ap1 : x);
      }
      break;
    case KACT_SOFTSIGN:
#pragma unroll
      for (int i = 0; i < N; i++)
        v[i] = v[i] * rcp_approx(1.0f + fabsf(v[i]));
      break;
    default: break;
  }
}

// ---- small helpers -------------------------------------------------------------------------
__device__ __forceinline__ float4 ld_ring(const float4* p)
{
  return __ldcg(p); // L2 only: ring lines are written by this CTA and re-read tiles later
}
__device__ __forceinline__ void st_ring(float4* p, const float4& v)
{
  __stcg(p, v);
}

// ---- tile-parallel hand-over (WaveNetKernelParams::tile_flags) -------------------------------
// A tile publishes "my ring columns of step k are in L2" by storing k + 1; its successor polls.
struct TileSync
{
  const int* prev; // flag of the same stream's previous tile (nullptr: nothing to wait for)
  int* mine; // this tile's flag (nullptr: classic mode)
  int tile_i; // index of this tile inside its stream (lock-step mode: tiles tile_i-1, tile_i-2, ... are polled)
};
__device__ __forceinline__ void tile_wait(const TileSync& ts, int step)
{
  if (ts.prev != nullptr) // uniform
  {
    if (threadIdx.x == 0)
    {
      int v;
      do
      {
        asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(ts.prev) : "memory");
      } while (v <= step);
    }
    __syncthreads();
  }
}
__device__ __forceinline__ void tile_publish(const TileSync& ts, int step)
{
  if (ts.mine != nullptr) // uniform
  {
    __threadfence(); // this thread's ring stores are visible device-wide
    __syncthreads();
    if (threadIdx.x == 0)
      asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(ts.mine), "r"(step + 1) : "memory");
  }
}

// ---- lock-step hand-over (WaveNetKernelParams::hist) ------------------------------------------
// "My columns of step `step` are in hist" (flag = step + 1), then wait until the `m` previous tiles of the stream
// have published the same step.  The first barrier also orders this CTA's own shared-tile writes before the reads
// that follow; lanes 0..m-1 poll one predecessor each.
constexpr int kLsFinalStep = 1 << 20;
// Spin on a flag with acquire loads.  (Relaxed loads in the loop plus one fence.acq_rel.gpu at the end -- to avoid the
// L1 invalidation each ld.acquire costs -- was slower: the fence waits for far more than the flag.)
__device__ __forceinline__ void ls_spin_until_above(const int* flag, const int step)
{
  int v;
  do
  {
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
  } while (v <= step);
}
__device__ __forceinline__ void ls_publish_wait(const TileSync& ts, const int step, const int m)
{
  // The CTA's hist stores are ordered before the barrier, the barrier before thread 0's release: the release is
  // cumulative over everything that happens-before it, so one fence (inside st.release.gpu) covers the whole CTA's
  // stores -- the pattern of a cooperative-groups grid barrier, cheaper than a __threadfence() per thread.
  __syncthreads();
  if (threadIdx.x == 0)
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(ts.mine), "r"(step + 1) : "memory");
  for (int k = threadIdx.x; k < m; k += blockDim.x)
    ls_spin_until_above(ts.mine - 1 - k, step);
  __syncthreads();
}

// ---- fp32 pairs ---------------------------------------------------------------------------------
// Accumulators and epilogue values are kept as 64-bit register pairs (two output channels, or two
// values of the element-wise math).  sm_90 has no packed FP32 arithmetic, so every pair operation is
// two scalar round-to-nearest instructions on the halves: the same numbers fma.rn.f32x2 /
// mul.rn.f32x2 / add.rn.f32x2 give, and ptxas keeps the halves in the register pair (no MOVs).
typedef unsigned long long u64;

__device__ __forceinline__ u64 pack2(const float lo, const float hi)
{
  u64 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void unpack2(const u64 v, float& lo, float& hi)
{
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ u64 tc_fma2(u64 a, u64 b, u64 c)
{
  float al, ah, bl, bh, cl, ch;
  unpack2(a, al, ah);
  unpack2(b, bl, bh);
  unpack2(c, cl, ch);
  return pack2(__fmaf_rn(al, bl, cl), __fmaf_rn(ah, bh, ch));
}
__device__ __forceinline__ u64 tc_mul2(u64 a, u64 b)
{
  float al, ah, bl, bh;
  unpack2(a, al, ah);
  unpack2(b, bl, bh);
  return pack2(__fmul_rn(al, bl), __fmul_rn(ah, bh));
}
__device__ __forceinline__ u64 tc_add2(u64 a, u64 b)
{
  float al, ah, bl, bh;
  unpack2(a, al, ah);
  unpack2(b, bl, bh);
  return pack2(__fadd_rn(al, bl), __fadd_rn(ah, bh));
}
__device__ __forceinline__ void fma2_acc(u64& acc, const u64 w, const u64 xx)
{
  acc = tc_fma2(w, xx, acc);
}
__device__ __forceinline__ void add2_acc(u64& acc, const u64 v)
{
  acc = tc_add2(acc, v);
}
__device__ __forceinline__ u64 tc_dup(float v)
{
  return pack2(v, v);
}
constexpr u64 kTcAbsMask = 0x7FFFFFFF7FFFFFFFull;
// the reference's rational fast_tanh (activations.h:91-98) on a pair
__device__ __forceinline__ u64 tc_fast_tanh2(u64 x)
{
  const u64 ax = x & kTcAbsMask;
  const u64 x2 = tc_mul2(x, x);
  const u64 c0 = tc_dup(2.45550750702956f);
  const u64 t1 = tc_fma2(tc_dup(0.821226666969744f), ax, tc_dup(0.893229853513558f));
  const u64 t0 = tc_fma2(c0, ax, c0);
  const u64 num = tc_mul2(x, tc_fma2(t1, x2, t0));
  const u64 s = tc_fma2(tc_dup(0.814642734961073f), tc_mul2(x, ax), x) & kTcAbsMask;
  const u64 d0 = tc_dup(2.44506634652299f);
  const u64 den = tc_fma2(tc_add2(x2, d0), s, d0);
  float dl, dh;
  unpack2(den, dl, dh);
  return tc_mul2(num, pack2(rcp_approx(dl), rcp_approx(dh)));
}

// acc[o] += w_row[o] * x for C outputs, two per register pair (x broadcast to both halves).
template <int C>
__device__ __forceinline__ void axpy_row(u64 (&acc)[C / 2], const float* __restrict__ w_row, const float x)
{
  const u64 xx = pack2(x, x);
#pragma unroll
  for (int q = 0; q < C / 4; q++)
  {
    const float4 w = *reinterpret_cast<const float4*>(w_row + 4 * q);
    fma2_acc(acc[2 * q], pack2(w.x, w.y), xx);
    fma2_acc(acc[2 * q + 1], pack2(w.z, w.w), xx);
  }
}

// One layer array for the S time steps a thread owns.
//   CIN  : channels of the array input (1 for the first array: the raw sample)
//   C    : channels == bottleneck (padded to a multiple of 4)
//   HOUT : rows of the head output (next array's C, or 1 for the last array)
//   LQ   : log2 of the frames per sub-tile.  (1 << LQ) == S * NT: the CTA's tile is one stream (long calls).
//          Smaller: the tile holds Q = S*NT >> LQ streams side by side, each with its own 64-column halo --
//          short calls (the reference tools' 64-frame blocks) are latency-bound per stream (20 layers x 2
//          barriers x ring loads), so several streams walk the layer chain together and share the weights.
//   state[j], Tv[j]: ring base and number of valid frames of the stream that owns this thread's j-th frame
//          (Tv[j] == 0 for a slot beyond the batch); stream0 locates the other sub-tiles' rings for the halo fill.
//   tabs0: absolute ring column of the tile's first frame, t_base + t0.  With a slot table (TBL) every stream's columns
//          are addressed from its own clock instead (WaveNetKernelParams::slots), re-read where they are used: the
//          streams of a tile need not share one.
//   LS   : lock-step tile-parallel mode (Q == 1 only): hist_a = this stream's history buffer at the array's first
//          plane, t0 = call-relative first frame of the tile (see WaveNetKernelParams::hist)
//   TBL  : the call carries a slot table (WaveNetKernelParams::slots); false compiles the table out entirely
template <int CIN, int C, int HOUT, int S, int NT, int LQ, bool LS, bool TBL>
__device__ __forceinline__ void array_forward(const WaveNetKernelParams& p, const ArrayDesc& A,
                                              const float* __restrict__ sw, float4* __restrict__ tile,
                                              float* const (&state)[S], const int stream0, const uint32_t tabs0,
                                              const TileSync& ts, const int step0, float4* const hist_a, const int t0,
                                              const int (&Tv)[S],
                                              const float (&hin)[S][CIN], const float (&cond)[S],
                                              u64 (&head)[S][C / 2], float (&hout)[S][C], float (&headout)[S][HOUT])
{
  constexpr int T = S * NT;
  constexpr int FQ = 1 << LQ; // frames per sub-tile
  constexpr int Q = T / FQ; // streams per tile
  constexpr int SW = kHalo + FQ; // columns of one sub-tile (halo + frames)
  constexpr int TW = Q * SW; // columns per plane in the shared tile
  constexpr int P = C / 4; // planes
  static_assert(Q >= 1 && Q * FQ == T && (Q == 1 || FQ <= NT), "sub-tile geometry");
  static_assert(!LS || Q == 1, "lock-step mode: one stream per tile");
  const int tid = threadIdx.x;
  const int NC = p.hist_cols; // LS: columns per plane of hist
  // this thread's j-th frame: sub-tile, frame inside it, tile column
  int fj[S], colj[S];
#pragma unroll
  for (int j = 0; j < S; j++)
  {
    const int trel = j * NT + tid;
    fj[j] = trel & (FQ - 1);
    colj[j] = (trel >> LQ) * SW + kHalo + fj[j];
  }
  constexpr int kColStep = (Q == 1) ? NT : (NT >> LQ) * SW; // colj[j] - colj[j-1]
  const int f_warp = (tid & (FQ - 1)) & ~31; // first frame of this warp inside its sub-tile (same for every j)
  auto sub_state = [&](int q) -> float* {
    const int s = min(stream0 + q, p.batch - 1);
    return p.state + (size_t)(TBL ? p.slots[s].stream : s) * p.state_stride;
  };
  // absolute ring column of frame t0 of sub-tile q's stream, and of the stream of this thread's j-th frame
  // (without a table both are tabs0: the table-free instantiation is the code of a handle-wide clock)
  auto sub_tabs = [&](int q) -> uint32_t {
    if constexpr (!TBL)
      return tabs0;
    const int s = min(stream0 + q, p.batch - 1);
    return p.slots[s].clock + (uint32_t)t0;
  };
  auto tabs_j = [&](int j) -> uint32_t {
    if constexpr (!TBL)
      return tabs0;
    return sub_tabs(Q == 1 ? 0 : (j * NT + tid) >> LQ);
  };

  // ---- rechannel (Conv1x1, no bias; model.cpp:492) -> this thread's columns of the tile
#pragma unroll
  for (int j = 0; j < S; j++)
  {
    u64 h[C / 2];
#pragma unroll
    for (int q = 0; q < C / 2; q++)
      h[q] = 0ull;
#pragma unroll
    for (int i = 0; i < CIN; i++)
      axpy_row<C>(h, sw + A.rech_off + i * C, hin[j][i]);
#pragma unroll
    for (int pl = 0; pl < P; pl++)
    {
      float4 v;
      unpack2(h[2 * pl], v.x, v.y);
      unpack2(h[2 * pl + 1], v.z, v.w);
      tile[pl * TW + colj[j]] = v;
      if constexpr (LS)
        if (fj[j] < Tv[j])
          st_ring(hist_a + (size_t)pl * NC + t0 + fj[j], v); // layer 0's input columns
    }
  }

#pragma unroll 1
  for (int li = 0; li < A.n_layers; li++)
  {
    // descriptor fields -> registers once per layer (they live in the kernel-parameter constant bank)
    const LayerDesc& Ld = p.layers[A.layer0 + li];
    const int K = Ld.kernel, dil = Ld.dilation, lookback = Ld.lookback;
    const uint32_t ring_mask = (uint32_t)Ld.ring_mask;
    const int R = Ld.ring_mask + 1;
    const float* __restrict__ w = sw + Ld.w_off;
    const float* __restrict__ w_bias = w + K * C * C;
    const float* __restrict__ w_mix = w_bias + C;
    const float* __restrict__ w_p = w_mix + C;
    const float* __restrict__ w_pb = w_p + C * C;
    const float* __restrict__ w_slopes = w_pb + C;
    float4* ring[S];
#pragma unroll
    for (int j = 0; j < S; j++)
      ring[j] = reinterpret_cast<float4*>(state[Q == 1 ? 0 : j] + Ld.ring_off);
    const int halo = (lookback <= kHalo) ? lookback : 0; // (a 64-column halo for the longer look-backs costs more than it saves: measured)

    // LS: this layer's input columns [call start, tile start) come from hist (written by the previous tiles during this
    // call), older ones from the ring
    const float4* const hist_l = LS ? hist_a + (size_t)li * P * NC : nullptr;
    if constexpr (LS)
      ls_publish_wait(ts, step0 + li, min(ts.tile_i, (lookback + FQ - 1) >> LQ));
    else
      tile_wait(ts, step0 + li); // tile-parallel mode: the previous tile's columns of this layer are in the ring

    // ---- phase 0: small-dilation layers pull their history [t0-L, t0) into the halo
    if constexpr (LS)
    {
      for (int idx = tid; idx < halo * P; idx += NT)
      {
        const int pl = idx / halo, col = idx - pl * halo;
        const int a = t0 - halo + col;
        tile[pl * TW + kHalo - halo + col] = ld_ring(
          a >= 0 ? hist_l + (size_t)pl * NC + a : ring[0] + pl * R + ((sub_tabs(0) - (uint32_t)halo + (uint32_t)col) & ring_mask));
      }
    }
    else if constexpr (Q == 1)
    {
      for (int idx = tid; idx < halo * P; idx += NT)
      {
        const int pl = idx / halo, col = idx - pl * halo;
        tile[pl * TW + kHalo - halo + col] =
          ld_ring(ring[0] + pl * R + ((sub_tabs(0) - (uint32_t)halo + (uint32_t)col) & ring_mask));
      }
    }
    else
    {
      for (int idx = tid; idx < Q * P * halo; idx += NT)
      {
        const int col = idx % halo, t2 = idx / halo;
        const int pl = t2 % P, q = t2 / P;
        const float4* __restrict__ rq = reinterpret_cast<const float4*>(sub_state(q) + Ld.ring_off);
        tile[pl * TW + q * SW + kHalo - halo + col] =
          ld_ring(rq + pl * R + ((sub_tabs(q) - (uint32_t)halo + (uint32_t)col) & ring_mask));
      }
    }
    if (!LS || halo > 0) // (LS: the hand-over's barrier already made the tile columns visible)
      __syncthreads(); // B0: tile columns (previous layer's phase 2) + halo are visible

    // ---- phase 1: z = b + M c + sum_k W_k h[t-(K-1-k)d] ; a = act(z) ; head += a
    u64 acc[S][C / 2];
#pragma unroll
    for (int j = 0; j < S; j++)
    {
#pragma unroll
      for (int q = 0; q < C / 4; q++)
      {
        const float4 b4 = *reinterpret_cast<const float4*>(w_bias + 4 * q);
        acc[j][2 * q] = pack2(b4.x, b4.y);
        acc[j][2 * q + 1] = pack2(b4.z, b4.w);
      }
      axpy_row<C>(acc[j], w_mix, cond[j]);
    }
    const float* __restrict__ w_row = w; // walks [k][in][out] linearly
#pragma unroll 1
    for (int k = 0; k < K; k++)
    {
      const int off = (K - 1 - k) * dil;
      // Warp-uniform fast path: every lane of this warp finds both of its frames in the shared tile (halo
      // included).  True for all warps of the small-dilation layers and for the later warps of a tile otherwise;
      // the loop below then carries no ring addressing at all (it was ~20 of 110 issued instructions per plane).
      if ((f_warp - off) >= -halo)
      {
        const float4* __restrict__ sp0 = tile + colj[0] - off;
#pragma unroll kPlUnroll
        for (int pl = 0; pl < P; pl++)
        {
          float4 xq[S];
#pragma unroll
          for (int j = 0; j < S; j++)
            xq[j] = sp0[pl * TW + j * kColStep];
#pragma unroll
          for (int i = 0; i < 4; i++)
          {
#pragma unroll
            for (int j = 0; j < S; j++)
            {
              const float xs = (i == 0) ? xq[j].x : (i == 1) ? xq[j].y : (i == 2) ? xq[j].z : xq[j].w;
              axpy_row<C>(acc[j], w_row, xs);
            }
            w_row += C;
          }
        }
        continue;
      }
      // general path: tap source per owned time step, resolved once per tap: the shared tile or the ring
      const float4* sp[S];
      uint32_t gi[S];
      bool glob[S];
      const float4* gp[S]; // LS: the column in hist (this call) or in the ring (before it), and its plane stride
      int gs[S];
#pragma unroll
      for (int j = 0; j < S; j++)
      {
        const int rel = fj[j] - off;
        glob[j] = rel < -halo;
        sp[j] = tile + colj[j] - off;
        gi[j] = (tabs_j(j) + (uint32_t)rel) & ring_mask;
        if constexpr (LS)
        {
          const bool in_call = t0 + rel >= 0;
          gp[j] = in_call ? hist_l + (t0 + rel) : ring[j] + gi[j];
          gs[j] = in_call ? NC : R;
        }
      }
#pragma unroll kPlUnroll
      for (int pl = 0; pl < P; pl++)
      {
        float4 xq[S];
#pragma unroll
        for (int j = 0; j < S; j++)
        {
          if constexpr (LS)
          {
            xq[j] = glob[j] ? ld_ring(gp[j]) : *sp[j];
            gp[j] += gs[j];
          }
          else if (glob[j])
            xq[j] = ld_ring(ring[j] + gi[j]);
          else
            xq[j] = *sp[j];
          sp[j] += TW;
          gi[j] += (uint32_t)R;
        }
#pragma unroll
        for (int i = 0; i < 4; i++)
        {
#pragma unroll
          for (int j = 0; j < S; j++)
          {
            const float xs = (i == 0) ? xq[j].x : (i == 1) ? xq[j].y : (i == 2) ? xq[j].z : xq[j].w;
            axpy_row<C>(acc[j], w_row, xs);
          }
          w_row += C;
        }
      }
    }
    float a[S][C];
#pragma unroll
    for (int j = 0; j < S; j++)
    {
      if (Ld.act == KACT_FASTTANH)
      {
        // the benchmark regime: the rational fast_tanh on packed pairs (7 instead of 11 issue slots per element)
#pragma unroll
        for (int q = 0; q < C / 2; q++)
        {
          acc[j][q] = tc_fast_tanh2(acc[j][q]);
          add2_acc(head[j][q], acc[j][q]); // model.cpp:530
          unpack2(acc[j][q], a[j][2 * q], a[j][2 * q + 1]);
        }
        continue;
      }
#pragma unroll
      for (int q = 0; q < C / 2; q++)
        unpack2(acc[j][q], a[j][2 * q], a[j][2 * q + 1]);
      apply_activation<C>(a[j], Ld, w_slopes);
#pragma unroll
      for (int q = 0; q < C / 2; q++)
        add2_acc(head[j][q], pack2(a[j][2 * q], a[j][2 * q + 1])); // model.cpp:530
    }
    __syncthreads(); // B1: every tap read of this layer's input is done

    // ---- phase 2: persist the tail of h_l, then h_{l+1} = h_l + p + P a  (model.cpp:243,376)
    const bool last = (li + 1 == A.n_layers);
    u64 hn[S][C / 2];
#pragma unroll
    for (int j = 0; j < S; j++)
    {
      const bool keep = !LS && (fj[j] < Tv[j]) && (fj[j] >= Tv[j] - lookback); // (LS: the rings are rewritten at the end)
#pragma unroll
      for (int pl = 0; pl < P; pl++)
      {
        const float4 own = tile[pl * TW + colj[j]];
        if (keep)
          st_ring(ring[j] + pl * R + ((tabs_j(j) + (uint32_t)fj[j]) & ring_mask), own);
        const float4 pb = *reinterpret_cast<const float4*>(w_pb + 4 * pl);
        hn[j][2 * pl] = pack2(own.x + pb.x, own.y + pb.y);
        hn[j][2 * pl + 1] = pack2(own.z + pb.z, own.w + pb.w);
      }
    }
#pragma unroll
    for (int i = 0; i < C; i++)
    {
      const float* __restrict__ p_row = w_p + i * C;
#pragma unroll
      for (int j = 0; j < S; j++)
        axpy_row<C>(hn[j], p_row, a[j][i]);
    }
#pragma unroll
    for (int j = 0; j < S; j++)
    {
      if (!last)
      {
#pragma unroll
        for (int pl = 0; pl < P; pl++)
        {
          float4 v;
          unpack2(hn[j][2 * pl], v.x, v.y);
          unpack2(hn[j][2 * pl + 1], v.z, v.w);
          tile[pl * TW + colj[j]] = v;
          if constexpr (LS)
            if (fj[j] < Tv[j])
              st_ring(hist_a + ((size_t)(li + 1) * P + pl) * NC + t0 + fj[j], v); // the next layer's input columns
        }
      }
      else
      {
#pragma unroll
        for (int q = 0; q < C / 2; q++)
          unpack2(hn[j][q], hout[j][2 * q], hout[j][2 * q + 1]);
      }
    }
    if constexpr (!LS)
      tile_publish(ts, step0 + li);
  }

  const float* __restrict__ wh = sw + A.head_off;
  if (A.head_kernel > 1)
  {
    // ---- head rechannel as a causal convolution over the head accumulator (A2 family: kernel 16;
    //      model.cpp:397-400,548): the accumulator columns go through the tile so that every thread can
    //      read its predecessors', the last (HK-1)*dilation columns of a stream live in the head ring
    const int HK = A.head_kernel, hdil = A.head_dilation, HL = (HK - 1) * hdil;
    const uint32_t hmask = (uint32_t)A.head_ring_mask;
    const int HR = A.head_ring_mask + 1;
    float4* const hist_h = LS ? hist_a + (size_t)A.n_layers * P * NC : nullptr; // LS: the head accumulator's columns
    if constexpr (!LS)
      tile_wait(ts, step0 + A.n_layers);
    float4* hring[S];
#pragma unroll
    for (int j = 0; j < S; j++)
      hring[j] = reinterpret_cast<float4*>(state[Q == 1 ? 0 : j] + A.head_ring_off);
    const float* __restrict__ w_hb = wh + HK * C * HOUT;
#pragma unroll
    for (int j = 0; j < S; j++)
#pragma unroll
      for (int pl = 0; pl < P; pl++)
      {
        float4 v;
        unpack2(head[j][2 * pl], v.x, v.y);
        unpack2(head[j][2 * pl + 1], v.z, v.w);
        tile[pl * TW + colj[j]] = v;
        if constexpr (LS)
          if (fj[j] < Tv[j])
            st_ring(hist_h + (size_t)pl * NC + t0 + fj[j], v);
      }
    if constexpr (LS)
    {
      ls_publish_wait(ts, step0 + A.n_layers, min(ts.tile_i, (HL + FQ - 1) >> LQ));
      for (int idx = tid; idx < P * HL; idx += NT)
      {
        const int pl = idx / HL, col = idx - pl * HL;
        const int a = t0 - HL + col;
        tile[pl * TW + kHalo - HL + col] =
          ld_ring(a >= 0 ? hist_h + (size_t)pl * NC + a : hring[0] + pl * HR + ((sub_tabs(0) - (uint32_t)HL + (uint32_t)col) & hmask));
      }
    }
    else
    {
      for (int idx = tid; idx < Q * P * HL; idx += NT)
      {
        const int col = idx % HL, t2 = idx / HL;
        const int pl = t2 % P, q = t2 / P;
        const float4* __restrict__ rq =
          (Q == 1) ? hring[0] : reinterpret_cast<const float4*>(sub_state(q) + A.head_ring_off);
        const uint32_t tq = sub_tabs(Q == 1 ? 0 : q);
        tile[pl * TW + q * SW + kHalo - HL + col] = ld_ring(rq + pl * HR + ((tq - (uint32_t)HL + (uint32_t)col) & hmask));
      }
    }
    __syncthreads(); // accumulator columns + halo visible; all ring reads done before the ring is rewritten
#pragma unroll
    for (int j = 0; j < S; j++)
    {
      if (!LS && (fj[j] < Tv[j]) && (fj[j] >= Tv[j] - HL))
      {
#pragma unroll
        for (int pl = 0; pl < P; pl++)
          st_ring(hring[j] + pl * HR + ((tabs_j(j) + (uint32_t)fj[j]) & hmask), tile[pl * TW + colj[j]]);
      }
      float out[HOUT];
#pragma unroll
      for (int ho = 0; ho < HOUT; ho++)
        out[ho] = w_hb[ho];
      const float* __restrict__ w_row = wh; // walks [k][in][HOUT] linearly
#pragma unroll 1
      for (int k = 0; k < HK; k++)
      {
        const float4* sp = tile + colj[j] - (HK - 1 - k) * hdil;
#pragma unroll
        for (int pl = 0; pl < P; pl++)
        {
          const float4 xq = sp[pl * TW];
          const float xs[4] = {xq.x, xq.y, xq.z, xq.w};
#pragma unroll
          for (int i = 0; i < 4; i++)
          {
#pragma unroll
            for (int ho = 0; ho < HOUT; ho++)
              out[ho] = fmaf(w_row[ho], xs[i], out[ho]);
            w_row += HOUT;
          }
        }
      }
#pragma unroll
      for (int ho = 0; ho < HOUT; ho++)
        headout[j][ho] = out[ho];
    }
    if constexpr (!LS)
      tile_publish(ts, step0 + A.n_layers);
    __syncthreads(); // the next array / tile rewrites the tile columns
    return;
  }

  // ---- head rechannel (kernel size 1; model.cpp:548): headout = H head (+ g)
#pragma unroll
  for (int j = 0; j < S; j++)
  {
    float hd[C];
#pragma unroll
    for (int q = 0; q < C / 2; q++)
      unpack2(head[j][q], hd[2 * q], hd[2 * q + 1]);
    if constexpr (HOUT == 1)
    {
      float s = 0.0f;
#pragma unroll
      for (int i = 0; i < C; i++)
        s = fmaf(wh[i], hd[i], s);
      headout[j][0] = s + wh[C];
    }
    else
    {
      u64 ho[HOUT / 2];
#pragma unroll
      for (int q = 0; q < HOUT / 4; q++)
      {
        const float4 g = *reinterpret_cast<const float4*>(wh + C * HOUT + 4 * q);
        ho[2 * q] = pack2(g.x, g.y);
        ho[2 * q + 1] = pack2(g.z, g.w);
      }
#pragma unroll
      for (int i = 0; i < C; i++)
        axpy_row<HOUT>(ho, wh + i * HOUT, hd[i]);
#pragma unroll
      for (int q = 0; q < HOUT / 2; q++)
        unpack2(ho[q], headout[j][2 * q], headout[j][2 * q + 1]);
    }
  }
}

// Lock-step mode epilogue: the stream's rings take the last `lookback` columns of the call from hist (every tile
// copies the columns it owns).  Runs after every tile of the stream has finished reading the rings.  TBL: n is the
// stream's own count from the slot table (without one the call's p.n_frames).
template <int C, int S, int NT, int LQ, bool TBL>
__device__ __forceinline__ void ls_write_back(const WaveNetKernelParams& p, const ArrayDesc& A, float* state,
                                              const float4* hist_a, const int t0, const uint32_t tabs0, const int tv,
                                              const int n)
{
  constexpr int P = C / 4;
  const int NC = p.hist_cols;
#pragma unroll 1
  for (int li = 0; li <= A.n_layers; li++)
  {
    int lookback, mask, off;
    if (li < A.n_layers)
    {
      const LayerDesc& Ld = p.layers[A.layer0 + li];
      lookback = Ld.lookback, mask = Ld.ring_mask, off = Ld.ring_off;
    }
    else
    {
      if (A.head_kernel <= 1)
        break;
      lookback = (A.head_kernel - 1) * A.head_dilation, mask = A.head_ring_mask, off = A.head_ring_off;
    }
    float4* ring = reinterpret_cast<float4*>(state + off);
    const float4* h = hist_a + (size_t)li * P * NC;
#pragma unroll
    for (int j = 0; j < S; j++)
    {
      const int f = (j * NT + (int)threadIdx.x) & ((1 << LQ) - 1);
      if (f < tv && t0 + f >= (TBL ? n : p.n_frames) - lookback)
      {
#pragma unroll
        for (int pl = 0; pl < P; pl++)
          st_ring(ring + pl * (mask + 1) + ((tabs0 + (uint32_t)f) & (uint32_t)mask), ld_ring(h + (size_t)pl * NC + t0 + f));
      }
    }
  }
}

// One persistent CTA per slot of Q = (S * NT) >> LQ streams.  C1 == 0: single layer array.
// LS: lock-step tile-parallel mode (one CTA per (stream, tile), see WaveNetKernelParams::hist); needs tile_flags.
// TBL: the call carries a slot table (a separate instantiation, so calls without one run exactly the table-free code).
template <int C0, int C1, int S, int NT, int MINB, int LQ, bool LS = false, bool TBL = false>
__global__ void __launch_bounds__(NT, MINB) wavenet_fused_kernel(const __grid_constant__ WaveNetKernelParams p)
{
  static_assert(!LS || (S * NT) == (1 << LQ), "lock-step mode: one stream per tile");
  constexpr int T = S * NT;
  constexpr int FQ = 1 << LQ;
  constexpr int Q = T / FQ;
  extern __shared__ float4 smem4[];
  float* sw = reinterpret_cast<float*>(smem4);
  float4* tile = smem4 + (p.n_weight_floats + 3) / 4;

  const int tid = threadIdx.x;
  // weights -> shared memory, once per CTA.  TBL: once per model the CTA meets (a bank's positions run their own models):
  // the blob is reloaded only when the next pass's model is not the one in shared memory.
  if constexpr (!TBL)
  {
    const float4* src = reinterpret_cast<const float4*>(p.weights);
    for (int i = tid; i < (p.n_weight_floats + 3) / 4; i += NT)
      smem4[i] = __ldg(src + i);
    __syncthreads();
  }
  int loaded = -1; // TBL: the model whose blob is in shared memory

  // classic mode: persistent CTA, slots of Q streams, all tiles of a call in turn.  Tile-parallel mode (Q == 1):
  // this CTA owns ONE (stream, tile) and hands its ring columns to the next tile's CTA layer by layer.
  int s_begin = blockIdx.x * Q, s_end = p.batch, s_step = gridDim.x * Q;
  int t_begin = 0, t_end = p.n_frames;
  TileSync ts{nullptr, nullptr, 0};
  if (Q == 1 && (LS || p.tile_flags != nullptr))
  {
    const int tile_i = blockIdx.x % p.tiles_per_stream;
    s_begin = blockIdx.x / p.tiles_per_stream;
    s_end = min(s_begin + 1, p.batch);
    t_begin = tile_i * FQ;
    t_end = min(p.n_frames, t_begin + FQ);
    ts.mine = p.tile_flags + (size_t)s_begin * p.tiles_per_stream + tile_i;
    ts.prev = tile_i > 0 ? ts.mine - 1 : nullptr;
    ts.tile_i = tile_i;
  }
  const int step1 = p.arrays[0].n_layers + 1; // first hand-over step of the second layer array

  for (int stream0 = s_begin; stream0 < s_end; stream0 += s_step)
  {
    // the stream each of this thread's frames belongs to (slots beyond the batch alias the last stream, masked by Tv)
    // (position sc of the call: state row from the slot table, or row sc; array_forward reads the clocks)
    auto position = [&](int j) -> int { return min(stream0 + ((Q == 1 ? 0 : j * NT + tid) >> LQ), p.batch - 1); };
    float* state[S];
    const float* xin[S];
    float* yout[S];
    bool live[S];
    int fj[S];
#pragma unroll
    for (int j = 0; j < S; j++)
    {
      const int trel = j * NT + tid;
      const int sj = stream0 + (trel >> LQ);
      live[j] = sj < p.batch;
      const size_t sc = (size_t)min(sj, p.batch - 1);
      const size_t row = TBL ? (size_t)p.slots[position(j)].stream : sc;
      state[j] = p.state + row * p.state_stride;
      xin[j] = p.in + sc * p.in_stride;
      yout[j] = p.out + sc * p.out_stride;
      fj[j] = trel & (FQ - 1);
    }
    // TBL: every position runs its own count of frames (slots[].frames <= p.n_frames).  Q == 1: the tiles stop at the
    // stream's count -- a tile-parallel CTA whose tile starts past it has no work, and no tile of the stream waits on it.
    // Q > 1: the slot's tiles run to its longest stream and a sub-tile past its stream's count gets Tv = 0, the masking
    // of a slot beyond the batch.
    // TBL, model banks: the slot runs one pass per distinct model among its positions (Q == 1: one pass).  A pass masks the
    // sub-tiles of the other models with Tv = 0 -- their state stays bit for bit -- so a homogeneous slot costs one pass.
    int n_all[S]; // frames of the stream of this thread's j-th frame (TBL only)
    unsigned todo = 0; // TBL: sub-tiles of the slot still to run
    if constexpr (TBL)
    {
#pragma unroll
      for (int j = 0; j < S; j++)
        n_all[j] = live[j] ? p.slots[position(j)].frames : 0;
#pragma unroll
      for (int q = 0; q < Q; q++)
        if (stream0 + q < p.batch)
          todo |= 1u << q;
    }
    do
    {
      int n_pos[S]; // TBL: n_all within this pass, 0 outside it
      int t_stop = t_end;
      float head_scale = p.head_scale;
      if constexpr (TBL)
      {
        const int mdl = p.slots[stream0 + __ffs(todo) - 1].model;
        unsigned pass = 0;
        int n_max = 0;
#pragma unroll
        for (int q = 0; q < Q; q++)
          if (((todo >> q) & 1u) && p.slots[stream0 + q].model == mdl)
          {
            pass |= 1u << q;
            n_max = max(n_max, p.slots[stream0 + q].frames);
          }
        todo &= ~pass;
#pragma unroll
        for (int j = 0; j < S; j++)
          n_pos[j] = ((pass >> ((Q == 1 ? 0 : j * NT + tid) >> LQ)) & 1u) ? n_all[j] : 0;
        t_stop = min(t_end, n_max);
        if (mdl != loaded && t_begin < t_stop) // (uniform: every thread reads the same table entries)
        {
          __syncthreads(); // the previous pass is done with the blob and the tile
          const float4* src = reinterpret_cast<const float4*>(p.weights + (size_t)mdl * p.weight_stride);
          for (int i = tid; i < (p.n_weight_floats + 3) / 4; i += NT)
            smem4[i] = __ldg(src + i);
          __syncthreads();
          loaded = mdl;
        }
        if (p.head_scales != nullptr)
          head_scale = p.head_scales[mdl];
      }

      for (int t0 = t_begin; t0 < t_stop; t0 += FQ)
      {
        const int tv = min(FQ, p.n_frames - t0);
        const uint32_t tabs0 = p.t_base + (uint32_t)t0;
        // LS: this stream's history buffer at the first plane of each array
        float4* const hist_s = LS ? reinterpret_cast<float4*>(p.hist + (size_t)stream0 * p.hist_stride) : nullptr;
        float4* const hist0 = LS ? hist_s + (size_t)p.hist_plane0[0] * p.hist_cols : nullptr;
        float4* const hist1 = LS ? hist_s + (size_t)p.hist_plane0[1] * p.hist_cols : nullptr;
        int Tv[S];
        float x[S][1], cond[S];
#pragma unroll
        for (int j = 0; j < S; j++)
        {
          if constexpr (TBL)
            Tv[j] = min(FQ, max(0, n_pos[j] - t0));
          else
            Tv[j] = live[j] ? tv : 0;
          x[j][0] = (fj[j] < Tv[j]) ? __ldg(xin[j] + t0 + fj[j]) : 0.0f;
          cond[j] = x[j][0]; // no condition_dsp: condition == input (model.cpp:781)
        }
        float y[S];
        if constexpr (C1 == 0)
        {
          u64 head0[S][C0 / 2];
#pragma unroll
          for (int j = 0; j < S; j++)
#pragma unroll
            for (int q = 0; q < C0 / 2; q++)
              head0[j][q] = 0ull; // model.cpp:469
          float hout0[S][C0], ho0[S][1];
          array_forward<1, C0, 1, S, NT, LQ, LS, TBL>(p, p.arrays[0], sw, tile, state, stream0, tabs0, ts, 0, hist0, t0, Tv, x, cond,
                                                 head0, hout0, ho0);
#pragma unroll
          for (int j = 0; j < S; j++)
            y[j] = ho0[j][0];
        }
        else
        {
          float hout0[S][C0], ho0[S][C1];
          {
            u64 head0[S][C0 / 2];
#pragma unroll
            for (int j = 0; j < S; j++)
#pragma unroll
              for (int q = 0; q < C0 / 2; q++)
                head0[j][q] = 0ull;
            array_forward<1, C0, C1, S, NT, LQ, LS, TBL>(p, p.arrays[0], sw, tile, state, stream0, tabs0, ts, 0, hist0, t0, Tv, x, cond,
                                                    head0, hout0, ho0);
          }
          // second array: layer input = previous array's layer output, head accumulator starts from
          // the previous array's head output (model.cpp:846-848, :473-486)
          u64 head1[S][C1 / 2];
#pragma unroll
          for (int j = 0; j < S; j++)
#pragma unroll
            for (int q = 0; q < C1 / 2; q++)
              head1[j][q] = pack2(ho0[j][2 * q], ho0[j][2 * q + 1]);
          float hout1[S][C1], ho1[S][1];
          array_forward<C0, C1, 1, S, NT, LQ, LS, TBL>(p, p.arrays[1], sw, tile, state, stream0, tabs0, ts, step1, hist1, t0, Tv, hout0,
                                                  cond, head1, hout1, ho1);
#pragma unroll
          for (int j = 0; j < S; j++)
            y[j] = ho1[j][0];
        }
#pragma unroll
        for (int j = 0; j < S; j++)
          if (fj[j] < Tv[j])
            yout[j][t0 + fj[j]] = head_scale * y[j]; // model.cpp:888-897
        if constexpr (LS)
        {
          // every tile of the stream is done with the rings -> rewrite them from hist for the next call.  (TBL: only the
          // stream's own tiles ever publish -- the tiles past its count have no work -- so the wait stops at them.)
          ls_publish_wait(ts, kLsFinalStep, 0);
          for (int k = tid; k < (TBL ? (n_pos[0] + FQ - 1) >> LQ : p.tiles_per_stream); k += NT)
            ls_spin_until_above(ts.mine - ts.tile_i + k, kLsFinalStep);
          __syncthreads();
          const uint32_t tabs_s = TBL ? p.slots[position(0)].clock + (uint32_t)t0 : tabs0;
          ls_write_back<C0, S, NT, LQ, TBL>(p, p.arrays[0], state[0], hist0, t0, tabs_s, Tv[0], n_pos[0]);
          if constexpr (C1 != 0)
            ls_write_back<C1, S, NT, LQ, TBL>(p, p.arrays[1], state[0], hist1, t0, tabs_s, Tv[0], n_pos[0]);
        }
      }
    } while (TBL && todo != 0);
    __syncthreads(); // the next streams reuse the tile
  }
}

} // namespace namb200
