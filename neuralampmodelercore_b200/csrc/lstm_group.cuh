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
//
// BANK (model banks, nam_b200_create_bank_*): the CTA's SPC streams may run different models.  Shared memory holds
// bank_copies padded copies (the host sizes them from the call's table: the most distinct models any CTA of the launch
// has, capped by what fits in 227 KB).  A CTA with more distinct models than copies makes one more pass over its chunk loop
// per bank_copies models; a group outside the pass steps with `step` false, exactly like a stream past its ragged count.
// A CTA of one model therefore costs one copy and one pass, as on an ordinary handle; round-robin binding of lstm.nam-sized
// models (76 floats a copy, all 32 copies fit) costs no extra pass, of H = 64 models (~17k floats, 3 copies of the 4 SPC
// fit) a second pass.  Each group's arithmetic is the ordinary instantiation's, on its own model's copy.
#pragma once

namespace namb200
{

constexpr int kLstmGroupThreads = 128;
constexpr int kLstmGroupChunk = 32; // frames staged per tile
constexpr int kLstmGroupMaxLayers = 4;
constexpr int kLstmGroupMaxHidden = 64; // two units per lane at G = 32

template <int G, bool BANK = false>
__global__ void __launch_bounds__(kLstmGroupThreads) lstm_group_kernel(const LstmKernelParams p)
{
  constexpr int SPC = kLstmGroupThreads / G; // streams per CTA
  constexpr int UPL = (G == 32) ? 2 : 1; // units per lane
  extern __shared__ float smem[];
  const int tid = threadIdx.x;
  const int H = p.hidden, L = p.num_layers;
  const int lane = tid % G, sl = tid / G; // lane in the group, stream slot in the CTA
  // shared: a model's copy -- per layer W rows padded to an odd stride | b[4H]; then head_w[H] | head_b -- (a bank:
  // bank_copies of them); then the I/O tiles
  float* sw = smem;
  int w_floats = 0;
  for (int l = 0; l < L; l++)
  {
    const int W = ((l == 0) ? p.input_size : H) + H;
    w_floats += 4 * H * (W | 1) + 4 * H;
  }
  const int copy_floats = w_floats + H + 1;
  const int n_copies = BANK ? p.bank_copies : 1;
  float* sio = sw + n_copies * copy_floats;
  float* sout = sio + SPC * (kLstmGroupChunk + 1);
  auto load_model = [&](const float* src, float* dst) {
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
      dst[i] = __ldg(src + i);
  };
  if constexpr (!BANK)
    load_model(p.weights, sw);

  const int stream = blockIdx.x * SPC + sl;
  const bool live = stream < p.batch;
  const size_t row = p.slots ? (size_t)p.slots[live ? stream : 0].stream : (size_t)stream; // state row of this position
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
        const float* st = p.state + row * p.state_stride + (size_t)l * 2 * H;
        h[l][k] = st[unit[k]];
        c[l][k] = st[H + unit[k]];
      }
    }
  const int stream0 = blockIdx.x * SPC;
  // BANK: the CTA's distinct models in order of first appearance (s_models, s_distinct of them) and the rank of each
  // position's model in that list (s_rank; -1 beyond the batch)
  __shared__ int s_models[BANK ? SPC : 1], s_rank[BANK ? SPC : 1], s_distinct;
  if constexpr (BANK)
  {
    if (tid < 32) // (SPC <= 32: warp 0 looks at every position)
    {
      const int mdl = (tid < SPC && stream0 + tid < p.batch) ? p.slots[stream0 + tid].model : -1;
      int first = tid;
      for (int s = 31; s >= 0; s--)
      {
        const int o = __shfl_sync(0xffffffffu, mdl, s);
        first = (s < tid && o == mdl) ? s : first;
      }
      const bool leads = mdl >= 0 && first == tid;
      const unsigned leaders = __ballot_sync(0xffffffffu, leads);
      const int rank = __popc(leaders & ((1u << first) - 1u));
      if (leads)
        s_models[rank] = mdl;
      if (tid < SPC)
        s_rank[tid] = mdl >= 0 ? rank : -1;
      if (tid == 0)
        s_distinct = __popc(leaders);
    }
  }
  __syncthreads();

  // Passes: an ordinary CTA makes one.  A bank's CTA makes one per bank_copies of its distinct models, those models'
  // blobs staged in the copies; a group whose model is not in the pass runs 0 frames in it -- it keeps (c, h) and writes
  // no output, like a stream past its ragged count.  A CTA of one model makes one pass over one copy.
  const int n_pass = BANK ? (s_distinct + n_copies - 1) / n_copies : 1;
  for (int pass = 0; pass < n_pass; pass++)
  {
    const int c0 = pass * n_copies; // rank of the model in copy 0
    if constexpr (BANK)
      for (int j = 0; j < n_copies && c0 + j < s_distinct; j++) // (the previous pass ended on a barrier)
        load_model(p.weights + (size_t)s_models[c0 + j] * p.weight_stride, sw + j * copy_floats);
    auto in_pass = [&](int s) -> bool { return !BANK || (s_rank[s] >= c0 && s_rank[s] < c0 + n_copies); };
    const float* wm = sw + ((BANK && in_pass(sl)) ? (s_rank[sl] - c0) * copy_floats : 0); // this group's model
    const float* hm = wm + w_floats; // its head
    // frames of the CTA's slot s (slot table: the stream's own count; 0 beyond the batch or outside the pass).  The chunk
    // loop below holds barriers and the groups' shuffles, so it runs to the pass's longest stream; a group whose stream
    // has ended steps without keeping (c, h).
    auto frames_of = [&](int s) -> int {
      const int b = stream0 + s;
      return (b >= p.batch || !in_pass(s)) ? 0 : p.slots ? p.slots[b].frames : p.n_frames;
    };
    int n_cta = 0;
    for (int s = 0; s < SPC; s++)
      n_cta = max(n_cta, frames_of(s));
    const int n_me = frames_of(sl);
    for (int t0 = 0; t0 < n_cta; t0 += kLstmGroupChunk)
    {
      const int tc = min(kLstmGroupChunk, n_cta - t0);
      for (int idx = tid; idx < SPC * kLstmGroupChunk; idx += kLstmGroupThreads)
      {
        const int s = idx / kLstmGroupChunk, f = idx - s * kLstmGroupChunk;
        float v = 0.0f;
        if (t0 + f < frames_of(s))
          v = __ldg(p.in + (size_t)(stream0 + s) * p.in_stride + t0 + f);
        sio[s * (kLstmGroupChunk + 1) + f] = v;
      }
      __syncthreads();
      for (int f = 0; f < tc; f++)
      {
        const bool step = t0 + f < n_me; // false: this group's stream has ended, its (c, h) stay as they are
        const float x = sio[sl * (kLstmGroupChunk + 1) + f];
        const float* w = wm;
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
            const float hn = lstm_sigmoid(go, p.fast_tanh) * lstm_tanh(cn, p.fast_tanh);
            c[l][k] = step ? cn : c[l][k];
            h[l][k] = step ? hn : h[l][k];
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
          y = fmaf(hm[j], v, y);
        }
        if (lane == 0)
          sout[sl * (kLstmGroupChunk + 1) + f] = y + hm[H];
      }
      __syncthreads();
      for (int idx = tid; idx < SPC * kLstmGroupChunk; idx += kLstmGroupThreads)
      {
        const int s = idx / kLstmGroupChunk, f = idx - s * kLstmGroupChunk;
        if (t0 + f < frames_of(s))
          p.out[(size_t)(stream0 + s) * p.out_stride + t0 + f] = sout[s * (kLstmGroupChunk + 1) + f];
      }
      __syncthreads();
    }
  }
  if (live)
  {
#pragma unroll
    for (int l = 0; l < kLstmGroupMaxLayers; l++)
#pragma unroll
      for (int k = 0; k < UPL; k++)
        if (l < L && owns[k])
        {
          float* st = p.state + row * p.state_stride + (size_t)l * 2 * H;
          st[unit[k]] = h[l][k];
          st[H + unit[k]] = c[l][k];
        }
  }
}

} // namespace namb200
