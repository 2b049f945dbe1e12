// lstm_spec.cuh -- the MODEL-SPECIALISED LSTM kernel for sm_90a (small cells: sum over layers of 4H(I+H) <= ~300 FMAs).
//
// Compiled per model by NVRTC (jit_spec.cpp) together with a generated header that defines namespace `spec`: H, L, I as
// constexpr and the weights as bit patterns read through spec::w(i).  What it computes (reference, under NAM/):
//   lstm.cpp:31-68   LSTMCell::process_   ifgo = W [x ; h] + b, c' = sig(f) c + sig(i) tanh(g), h' = sig(o) tanh(c')
//   lstm.cpp:136-168 LSTM::_process_sample layer chain + head dot product
// in both activation regimes (lstm.cpp:48 reads the fast-tanh switch at run time: two kernels in the cubin).
//
// The recurrence is serial in time: throughput = streams in flight / latency of one step.  The lane-group kernel
// (lstm_group.cuh) pays, per step, shuffles for h, shared-memory loads for the weights and a run-time switch per
// activation: ~980 cycles per step for the H = 3 cell of lstm.nam.  Here ONE THREAD owns a stream, every loop is
// unrolled over compile-time H / L / I, every weight is an FFMA immediate and (h, c) are plain registers: a step is
// just its dependent chain -- 1 + H FMAs per gate, the activations, the cell update.  Audio goes through a
// [32 streams][32 frames] shared tile so that global loads and stores are 128-byte rows although each lane walks its
// own stream; the next tile's loads are issued a whole tile ahead.
//
// State layout == lstm_group.cuh / lstm_kernel: per stream, per layer h[H] | c[H] floats, so the kernels can be mixed.
#pragma once

#ifndef NAMB200_LSTM_SPEC_HEADER_INCLUDED
#error "include the generated model header (namespace spec) before lstm_spec.cuh"
#endif

namespace namb200_lstm_spec
{

struct LstmSpecParams
{
  float* state; // [batch][state_stride]
  long state_stride;
  const float* in; // [batch][in_stride]
  float* out;
  long in_stride, out_stride;
  int batch, n_frames;
};

__device__ __forceinline__ float rcp_approx(float x)
{
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
// activations.h:91-98 (same expression as namb200::act_fast_tanh)
__device__ __forceinline__ float fast_tanh(float x)
{
  const float ax = fabsf(x);
  const float x2 = x * x;
  const float num = x * (2.45550750702956f + 2.45550750702956f * ax + (0.893229853513558f + 0.821226666969744f * ax) * x2);
  const float den = 2.44506634652299f + (2.44506634652299f + x2) * fabsf(x + 0.814642734961073f * x * ax);
  return num * rcp_approx(den);
}
template <bool FAST>
__device__ __forceinline__ float sig(float x)
{
  if constexpr (FAST)
    return 0.5f * (fast_tanh(x * 0.5f) + 1.0f); // activations.h:100-103
  else
    return rcp_approx(1.0f + expf(-x)); // activations.h:64-67
}
template <bool FAST>
__device__ __forceinline__ float tnh(float x)
{
  if constexpr (FAST)
    return fast_tanh(x);
  else
    return tanhf(x);
}

constexpr int kTile = 32; // streams per CTA (one warp) == frames per staged tile

// float offset of layer l's W[4H][I_l + H] | b[4H]
__host__ __device__ constexpr int layer_offset(int l)
{
  int off = 0;
  for (int k = 0; k < l; k++)
    off += 4 * spec::H * ((k == 0 ? spec::I : spec::H) + spec::H) + 4 * spec::H;
  return off;
}

template <bool FAST>
__device__ __forceinline__ void lstm_spec_body(const LstmSpecParams& p)
{
  constexpr int H = spec::H, L = spec::L, I = spec::I;
  static_assert(I == 1, "mono models");
  __shared__ float sin_[kTile][kTile + 1];
  __shared__ float sout[kTile][kTile + 1];
  const int lane = threadIdx.x;
  const int stream0 = blockIdx.x * kTile;
  const int stream = stream0 + lane;
  const bool live = stream < p.batch;

  float h[L][H], c[L][H];
#pragma unroll
  for (int l = 0; l < L; l++)
#pragma unroll
    for (int u = 0; u < H; u++)
    {
      const float* st = p.state + (size_t)min(stream, p.batch - 1) * p.state_stride + l * 2 * H;
      h[l][u] = st[u];
      c[l][u] = st[H + u];
    }

  // tile loads: row r = stream stream0 + r, lane = frame; issued one tile ahead (registers), parked in shared memory
  float pre[kTile];
  auto fetch = [&](int t0) {
#pragma unroll
    for (int r = 0; r < kTile; r++)
    {
      const int s = stream0 + r;
      pre[r] = (s < p.batch && t0 + lane < p.n_frames) ? __ldg(p.in + (size_t)s * p.in_stride + t0 + lane) : 0.0f;
    }
  };
  fetch(0);
  for (int t0 = 0; t0 < p.n_frames; t0 += kTile)
  {
    const int tc = min(kTile, p.n_frames - t0);
    __syncwarp();
#pragma unroll
    for (int r = 0; r < kTile; r++)
      sin_[r][lane] = pre[r];
    __syncwarp();
    if (t0 + kTile < p.n_frames)
      fetch(t0 + kTile);
    for (int f = 0; f < tc; f++)
    {
      const float x = sin_[lane][f];
      float xin[H > I ? H : I];
      xin[0] = x;
#pragma unroll
      for (int l = 0; l < L; l++)
      {
        const int Il = (l == 0) ? I : H;
        const int W = Il + H;
        const int w0 = layer_offset(l), b0 = w0 + 4 * H * W;
        // ifgo = W [x ; h] + b   (lstm.cpp:36-40): rows i, f, g, o; input part first, then the bias.
        // Fast regime: fast_sigmoid(z) = 0.5 fast_tanh(0.5 z) + 0.5 (activations.h:100-103); the 0.5 z of the three
        // sigmoid gates is folded into their weights and biases (a power of two: bit-exact).
        float g[4 * H];
#pragma unroll
        for (int q = 0; q < 4; q++)
#pragma unroll
          for (int u = 0; u < H; u++)
          {
            const float sc = (FAST && q != 2) ? 0.5f : 1.0f;
            float a = 0.0f;
#pragma unroll
            for (int j = 0; j < Il; j++)
              a = fmaf(sc * spec::w(w0 + (q * H + u) * W + j), xin[j], a);
#pragma unroll
            for (int j = 0; j < H; j++)
              a = fmaf(sc * spec::w(w0 + (q * H + u) * W + Il + j), h[l][j], a);
            g[q * H + u] = a + sc * spec::w(b0 + q * H + u);
          }
        if constexpr (FAST)
        {
          // scalar on purpose: a lone warp per scheduler is bound by the dependent chain, which pairing the activations
          // does not shorten
#pragma unroll
          for (int u = 0; u < H; u++)
          {
            const float si = fmaf(0.5f, fast_tanh(g[u]), 0.5f), sf = fmaf(0.5f, fast_tanh(g[H + u]), 0.5f);
            const float cn = sf * c[l][u] + si * fast_tanh(g[2 * H + u]); // lstm.cpp:50-53
            c[l][u] = cn;
            h[l][u] = fmaf(0.5f, fast_tanh(g[3 * H + u]), 0.5f) * fast_tanh(cn); // :55-57
          }
        }
        else
        {
#pragma unroll
          for (int u = 0; u < H; u++)
          {
            const float cn = sig<false>(g[H + u]) * c[l][u] + sig<false>(g[u]) * tnh<false>(g[2 * H + u]); // lstm.cpp:61-63
            c[l][u] = cn;
            h[l][u] = sig<false>(g[3 * H + u]) * tnh<false>(cn); // :65-66
          }
        }
#pragma unroll
        for (int u = 0; u < H; u++)
          xin[u] = h[l][u];
      }
      // head (lstm.cpp:164-167)
      constexpr int hw = layer_offset(L);
      float y = 0.0f;
#pragma unroll
      for (int j = 0; j < H; j++)
        y = fmaf(spec::w(hw + j), h[L - 1][j], y);
      sout[lane][f] = y + spec::w(hw + H);
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < kTile; r++)
    {
      const int s = stream0 + r;
      if (s < p.batch && lane < tc)
        p.out[(size_t)s * p.out_stride + t0 + lane] = sout[r][lane];
    }
  }
  if (live)
  {
#pragma unroll
    for (int l = 0; l < L; l++)
#pragma unroll
      for (int u = 0; u < H; u++)
      {
        float* st = p.state + (size_t)stream * p.state_stride + l * 2 * H;
        st[u] = h[l][u];
        st[H + u] = c[l][u];
      }
  }
}

// ---- gate-split variant: FOUR lanes per stream, lane q = gate q (i, f, g, o) ----------------------------------------------
// One thread per stream issues ~290 instructions per step from a single warp per scheduler; the step's dependent chain is
// only ~150 cycles.  Here lane q of a group of four computes gate q's H
// pre-activations (its rows of W in registers: the rows differ per lane, so they cannot be immediates) and their
// activation; the 4H activated values are exchanged by shuffles and every lane updates (c, h) of all units redundantly,
// so nothing has to be broadcast back: ~115 instructions per lane per step, 8 streams per warp.
template <bool FAST>
__device__ __forceinline__ void lstm_gate_split_body(const LstmSpecParams& p)
{
  constexpr int H = spec::H, L = spec::L, I = spec::I;
  static_assert(I == 1, "mono models");
  constexpr int SPW = 8; // streams per warp
  __shared__ float sin_[SPW][kTile + 1];
  __shared__ float sout[SPW][kTile + 1];
  const int lane = threadIdx.x;
  const int q = lane & 3, grp = lane >> 2;
  const int stream0 = blockIdx.x * SPW;
  const int stream = stream0 + grp;
  const bool live = stream < p.batch;
  const unsigned base_lane = (unsigned)(lane & ~3);

  // my gate's rows: W[q*H + u][0 .. I+H) and b[q*H + u].  Fast regime: the 0.5 z of the sigmoid gates is folded in.
  const float sc = (FAST && q != 2) ? 0.5f : 1.0f;
  float wx[L][H], wh[L][H][H], wb[L][H];
#pragma unroll
  for (int l = 0; l < L; l++)
  {
    const int Il = (l == 0) ? I : H, W = Il + H;
    const int w0 = layer_offset(l), b0 = w0 + 4 * H * W;
#pragma unroll
    for (int u = 0; u < H; u++)
    {
      // (layer 0: one input column; deeper layers: H input columns, kept in wh2 below)
      wx[l][u] = (l == 0) ? sc * spec::w(w0 + (q * H + u) * W) : 0.0f;
#pragma unroll
      for (int j = 0; j < H; j++)
        wh[l][u][j] = sc * spec::w(w0 + (q * H + u) * W + Il + j);
      wb[l][u] = sc * spec::w(b0 + q * H + u);
    }
  }
  float wi[L > 1 ? L - 1 : 1][H][H]; // input part of layers 1.. (their input is the previous layer's h)
#pragma unroll
  for (int l = 1; l < L; l++)
  {
    const int W = 2 * H, w0 = layer_offset(l);
#pragma unroll
    for (int u = 0; u < H; u++)
#pragma unroll
      for (int j = 0; j < H; j++)
        wi[l - 1][u][j] = sc * spec::w(w0 + (q * H + u) * W + j);
  }
  // post-activation map: tanh gate t -> t; sigmoid gates (fast regime) t -> 0.5 t + 0.5
  const float ka = (FAST && q != 2) ? 0.5f : 1.0f, kb = (FAST && q != 2) ? 0.5f : 0.0f;

  float h[L][H], c[L][H];
#pragma unroll
  for (int l = 0; l < L; l++)
#pragma unroll
    for (int u = 0; u < H; u++)
    {
      const float* st = p.state + (size_t)min(stream, p.batch - 1) * p.state_stride + l * 2 * H;
      h[l][u] = st[u];
      c[l][u] = st[H + u];
    }

  for (int t0 = 0; t0 < p.n_frames; t0 += kTile)
  {
    const int tc = min(kTile, p.n_frames - t0);
    __syncwarp();
#pragma unroll
    for (int r = 0; r < SPW; r++)
    {
      const int s = stream0 + r;
      sin_[r][lane] = (s < p.batch && t0 + lane < p.n_frames) ? __ldg(p.in + (size_t)s * p.in_stride + t0 + lane) : 0.0f;
    }
    __syncwarp();
    for (int f = 0; f < tc; f++)
    {
      const float x = sin_[grp][f];
#pragma unroll
      for (int l = 0; l < L; l++)
      {
        // my gate's H pre-activations (lstm.cpp:36-40; input part first, then the recurrent part, then the bias)
        float g[H];
#pragma unroll
        for (int u = 0; u < H; u++)
        {
          float a = 0.0f;
          if (l == 0)
            a = fmaf(wx[0][u], x, a);
          else
          {
#pragma unroll
            for (int j = 0; j < H; j++)
              a = fmaf(wi[l > 0 ? l - 1 : 0][u][j], h[l > 0 ? l - 1 : 0][j], a);
          }
#pragma unroll
          for (int j = 0; j < H; j++)
            a = fmaf(wh[l][u][j], h[l][j], a);
          a += wb[l][u];
          if constexpr (FAST)
            g[u] = fmaf(ka, fast_tanh(a), kb);
          else
            g[u] = (q == 2) ? tanhf(a) : sig<false>(a);
        }
        // everybody gets all four gates of every unit, then updates (c, h) of all units
#pragma unroll
        for (int u = 0; u < H; u++)
        {
          const float gi = __shfl_sync(0xffffffffu, g[u], base_lane + 0), gf = __shfl_sync(0xffffffffu, g[u], base_lane + 1);
          const float gg = __shfl_sync(0xffffffffu, g[u], base_lane + 2), go = __shfl_sync(0xffffffffu, g[u], base_lane + 3);
          const float cn = gf * c[l][u] + gi * gg; // lstm.cpp:50-53,61-63
          c[l][u] = cn;
          h[l][u] = go * tnh<FAST>(cn); // :55-57,65-66
        }
      }
      // head (lstm.cpp:164-167)
      constexpr int hw = layer_offset(L);
      float y = 0.0f;
#pragma unroll
      for (int j = 0; j < H; j++)
        y = fmaf(spec::w(hw + j), h[L - 1][j], y);
      if (q == 0)
        sout[grp][f] = y + spec::w(hw + H);
    }
    __syncwarp();
#pragma unroll
    for (int r = 0; r < SPW; r++)
    {
      const int s = stream0 + r;
      if (s < p.batch && lane < tc)
        p.out[(size_t)s * p.out_stride + t0 + lane] = sout[r][lane];
    }
  }
  if (live && q == 0)
  {
#pragma unroll
    for (int l = 0; l < L; l++)
#pragma unroll
      for (int u = 0; u < H; u++)
      {
        float* st = p.state + (size_t)stream * p.state_stride + l * 2 * H;
        st[u] = h[l][u];
        st[H + u] = c[l][u];
      }
  }
}

} // namespace namb200_lstm_spec

extern "C" __global__ void __launch_bounds__(32) lstm_spec_kernel_exact(const __grid_constant__ namb200_lstm_spec::LstmSpecParams p)
{
  namb200_lstm_spec::lstm_spec_body<false>(p);
}
extern "C" __global__ void __launch_bounds__(32) lstm_spec_kernel_fast(const __grid_constant__ namb200_lstm_spec::LstmSpecParams p)
{
  namb200_lstm_spec::lstm_spec_body<true>(p);
}
// gate-split variants: 8 streams per 32-thread CTA
extern "C" __global__ void __launch_bounds__(32) lstm_spec_gates_kernel_exact(const __grid_constant__ namb200_lstm_spec::LstmSpecParams p)
{
  namb200_lstm_spec::lstm_gate_split_body<false>(p);
}
extern "C" __global__ void __launch_bounds__(32) lstm_spec_gates_kernel_fast(const __grid_constant__ namb200_lstm_spec::LstmSpecParams p)
{
  namb200_lstm_spec::lstm_gate_split_body<true>(p);
}
