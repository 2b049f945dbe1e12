// lstm_group.cuh -- LSTM recurrence with the units of a cell spread over a group of lanes
// (reference: NAM/lstm.cpp:31-68 LSTMCell::process_, :136-168 LSTM::_process_sample).
//
// The recurrence is serial in time, so throughput = streams in flight / latency of one step.  A thread per stream
// (lstm_kernel in nam_b200.cu, kept as the fallback for hidden sizes above 64) leaves most of the GPU idle at 4096
// streams and walks the whole 4H x (I+H) matvec plus 5H activations in one dependent chain.  Here a group of
// G = 4 / 8 / 16 / 32 lanes (the next power of two >= H, at most 32) owns a stream: lane u computes the four gate
// pre-activations of hidden unit u (and u + 32 when H > 32), reads the other units' h through warp shuffles and
// applies the five activations of its own unit -- a step costs 4(I+H) FMAs + (I+H) shuffles + 5 activations per
// lane instead of H times that, and there are G times more warps to schedule.  Weights sit in shared memory with an
// odd row stride (lane u reads row g*H+u: conflict-free); h and c never leave registers between frames.
#pragma once

namespace namb200
{

constexpr int kLstmGroupThreads = 128;
constexpr int kLstmGroupChunk = 32; // frames staged per tile
constexpr int kLstmGroupMaxLayers = 4;
constexpr int kLstmGroupMaxHidden = 64; // two units per lane at G = 32

template <int G>
__global__ void __launch_bounds__(kLstmGroupThreads) lstm_group_kernel(const LstmKernelParams p)
{
  constexpr int SPC = kLstmGroupThreads / G; // streams per CTA
  constexpr int UPL = (G == 32) ? 2 : 1; // units per lane
  extern __shared__ float smem[];
  const int tid = threadIdx.x;
  const int H = p.hidden, L = p.num_layers;
  const int lane = tid % G, sl = tid / G; // lane in the group, stream slot in the CTA
  // shared: per layer W rows padded to an odd stride | b[4H]; then head_w[H] | head_b; then the I/O tiles
  float* sw = smem;
  int w_floats = 0;
  for (int l = 0; l < L; l++)
  {
    const int W = ((l == 0) ? p.input_size : H) + H;
    w_floats += 4 * H * (W | 1) + 4 * H;
  }
  float* shead = sw + w_floats;
  float* sio = shead + H + 1;
  float* sout = sio + SPC * (kLstmGroupChunk + 1);
  {
    const float* src = p.weights;
    float* dst = sw;
    for (int l = 0; l < L; l++)
    {
      const int W = ((l == 0) ? p.input_size : H) + H, Wp = W | 1;
      for (int i = tid; i < 4 * H * W; i += kLstmGroupThreads)
        dst[(i / W) * Wp + (i % W)] = __ldg(src + i);
      for (int i = tid; i < 4 * H; i += kLstmGroupThreads)
        dst[4 * H * Wp + i] = __ldg(src + 4 * H * W + i);
      src += 4 * H * W + 4 * H;
      dst += 4 * H * Wp + 4 * H;
    }
    for (int i = tid; i < H + 1; i += kLstmGroupThreads)
      shead[i] = __ldg(src + i);
  }

  const int stream = blockIdx.x * SPC + sl;
  const bool live = stream < p.batch;
  // this lane's units (clamped: surplus lanes shadow the last unit and are never read)
  int unit[UPL];
  bool owns[UPL];
#pragma unroll
  for (int k = 0; k < UPL; k++)
  {
    owns[k] = lane + k * G < H;
    unit[k] = min(lane + k * G, H - 1);
  }
  float h[kLstmGroupMaxLayers][UPL], c[kLstmGroupMaxLayers][UPL];
#pragma unroll
  for (int l = 0; l < kLstmGroupMaxLayers; l++)
#pragma unroll
    for (int k = 0; k < UPL; k++)
    {
      h[l][k] = 0.0f;
      c[l][k] = 0.0f;
      if (l < L && live)
      {
        const float* st = p.state + (size_t)stream * p.state_stride + (size_t)l * 2 * H;
        h[l][k] = st[unit[k]];
        c[l][k] = st[H + unit[k]];
      }
    }
  __syncthreads();

  const int stream0 = blockIdx.x * SPC;
  for (int t0 = 0; t0 < p.n_frames; t0 += kLstmGroupChunk)
  {
    const int tc = min(kLstmGroupChunk, p.n_frames - t0);
    for (int idx = tid; idx < SPC * kLstmGroupChunk; idx += kLstmGroupThreads)
    {
      const int s = idx / kLstmGroupChunk, f = idx - s * kLstmGroupChunk;
      float v = 0.0f;
      if (stream0 + s < p.batch && f < tc)
        v = __ldg(p.in + (size_t)(stream0 + s) * p.in_stride + t0 + f);
      sio[s * (kLstmGroupChunk + 1) + f] = v;
    }
    __syncthreads();
    for (int f = 0; f < tc; f++)
    {
      const float x = sio[sl * (kLstmGroupChunk + 1) + f];
      const float* w = sw;
      float hl[UPL] = {}; // the last layer's new h
#pragma unroll
      for (int l = 0; l < kLstmGroupMaxLayers; l++)
      {
        if (l >= L)
          break;
        const int I = (l == 0) ? p.input_size : H;
        const int Wp = (I + H) | 1;
        const float* b = w + 4 * H * Wp;
        float acc[UPL][4];
#pragma unroll
        for (int k = 0; k < UPL; k++)
#pragma unroll
          for (int g = 0; g < 4; g++)
            acc[k][g] = 0.0f;
        // ifgo = W [x ; h] + b   (lstm.cpp:36-40); rows ordered i, f, g, o; input part first, like the reference
        if (l == 0)
        {
#pragma unroll
          for (int k = 0; k < UPL; k++)
#pragma unroll
            for (int g = 0; g < 4; g++)
              acc[k][g] = fmaf(w[(g * H + unit[k]) * Wp], x, acc[k][g]); // input_size == 1 on this path
        }
        else
        {
          for (int j = 0; j < I; j++)
          {
            const float v = __shfl_sync(0xffffffffu, (UPL == 2 && j >= G) ? h[l - 1][UPL - 1] : h[l - 1][0], j % G, G);
#pragma unroll
            for (int k = 0; k < UPL; k++)
#pragma unroll
              for (int g = 0; g < 4; g++)
                acc[k][g] = fmaf(w[(g * H + unit[k]) * Wp + j], v, acc[k][g]);
          }
        }
        for (int j = 0; j < H; j++)
        {
          const float v = __shfl_sync(0xffffffffu, (UPL == 2 && j >= G) ? h[l][UPL - 1] : h[l][0], j % G, G);
#pragma unroll
          for (int k = 0; k < UPL; k++)
#pragma unroll
            for (int g = 0; g < 4; g++)
              acc[k][g] = fmaf(w[(g * H + unit[k]) * Wp + I + j], v, acc[k][g]);
        }
        // every lane has read the old h of this layer: update (lstm.cpp:50-57 fast | :61-66 exact)
#pragma unroll
        for (int k = 0; k < UPL; k++)
        {
          const float gi = acc[k][0] + b[unit[k]], gf = acc[k][1] + b[H + unit[k]];
          const float gg = acc[k][2] + b[2 * H + unit[k]], go = acc[k][3] + b[3 * H + unit[k]];
          const float cn = lstm_sigmoid(gf, p.fast_tanh) * c[l][k] + lstm_sigmoid(gi, p.fast_tanh) * lstm_tanh(gg, p.fast_tanh);
          c[l][k] = cn;
          h[l][k] = lstm_sigmoid(go, p.fast_tanh) * lstm_tanh(cn, p.fast_tanh);
          if (l == L - 1)
            hl[k] = h[l][k];
        }
        w = b + 4 * H;
      }
      // head (lstm.cpp:164-167): sum over the group's units, in unit order like the reference's dot product
      float y = 0.0f;
      for (int j = 0; j < H; j++)
      {
        const float v = __shfl_sync(0xffffffffu, (UPL == 2 && j >= G) ? hl[UPL - 1] : hl[0], j % G, G);
        y = fmaf(shead[j], v, y);
      }
      if (lane == 0)
        sout[sl * (kLstmGroupChunk + 1) + f] = y + shead[H];
    }
    __syncthreads();
    for (int idx = tid; idx < SPC * kLstmGroupChunk; idx += kLstmGroupThreads)
    {
      const int s = idx / kLstmGroupChunk, f = idx - s * kLstmGroupChunk;
      if (stream0 + s < p.batch && f < tc)
        p.out[(size_t)(stream0 + s) * p.out_stride + t0 + f] = sout[s * (kLstmGroupChunk + 1) + f];
    }
    __syncthreads();
  }
  if (live)
  {
#pragma unroll
    for (int l = 0; l < kLstmGroupMaxLayers; l++)
#pragma unroll
      for (int k = 0; k < UPL; k++)
        if (l < L && owns[k])
        {
          float* st = p.state + (size_t)stream * p.state_stride + (size_t)l * 2 * H;
          st[unit[k]] = h[l][k];
          st[H + unit[k]] = c[l][k];
        }
  }
}

} // namespace namb200
