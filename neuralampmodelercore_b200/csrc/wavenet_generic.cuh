// wavenet_generic.cuh -- the general WaveNet kernel: every option of the reference's WaveNet
// (NAM/wavenet/model.cpp:183-393 Layer::Process, :463-549 LayerArray, :777-910 WaveNet::process with
// condition_dsp and the post-stack head :19-103; NAM/film.h:76-190; NAM/gating_activations.h:100-113,209-227),
// driven by the descriptors of generic_desc.h.
//
// One CTA per stream, one thread per frame of a 128-frame tile, the whole network layer by layer for the tile
// (the net is feed-forward, so the frames of a call are independent within a layer -- the same reframing as the
// fused kernel, without its specialisations): all vectors of a frame live in the owning thread's scratch, only the
// dilated taps cross threads, through the convolution's input ring in HBM/L2 (write the tile's columns, barrier,
// read the taps, barrier).  The models that need this path are small (example_models/wavenet_a2_max.nam:
// 818 + 1,052 weights) and exist for their features; the throughput families have the fused kernels.  Weights are
// staged in shared memory (transposed, four outputs per float4) and read at warp-uniform addresses.
#pragma once

#include "generic_desc.h"
#include "wavenet_fused.cuh" // activations

namespace namb200
{

struct GenThread
{
  const float* __restrict__ w;
  float* __restrict__ st; // this CTA's stream
  uint32_t t; // absolute index of this thread's frame
  bool valid; // the frame exists (threads beyond the end of a call still take part in the barriers)
};

__device__ __forceinline__ float g_act1(const GenThread& c, const GAct& A, float x, int ch)
{
  switch (A.type)
  {
    case KACT_TANH: return tanhf(x);
    case KACT_FASTTANH: return act_fast_tanh(x);
    case KACT_HARDTANH: return fminf(fmaxf(x, -1.0f), 1.0f);
    case KACT_RELU: return x > 0.0f ? x : 0.0f;
    case KACT_LEAKYRELU: return x > 0.0f ? x : A.p0 * x;
    case KACT_PRELU: return x > 0.0f ? x : c.w[A.slopes_off + (A.n_slopes == 1 ? 0 : ch)] * x;
    case KACT_SIGMOID: return act_sigmoid(x);
    case KACT_SILU: return x * act_sigmoid(x);
    case KACT_HARDSWISH:
    {
      const float t = x + 3.0f;
      const float cl = t < 0.0f ? 0.0f : (t > 6.0f ? 6.0f : t);
      return x * cl * (1.0f / 6.0f);
    }
    case KACT_LEAKYHARDTANH: return x < A.p0 ? (x - A.p0) * A.p2 + A.p0 : (x > A.p1 ? (x - A.p1) * A.p3 + A.p1 : x);
    case KACT_SOFTSIGN: return x * rcp_approx(1.0f + fabsf(x));
    default: return x;
  }
}

// out[i] = act(in[i]) for i < n, the activation chosen ONCE for the vector (the per-element switch of g_act1 cost
// more issue slots than the activation itself on the narrow models this kernel serves); in-place allowed
__device__ __forceinline__ void g_act_vec(const GenThread& c, const GAct& A, const float* in, float* out, const int n)
{
  switch (A.type)
  {
    case KACT_TANH:
      for (int i = 0; i < n; i++)
        out[i] = tanhf(in[i]);
      break;
    case KACT_FASTTANH:
      for (int i = 0; i < n; i++)
        out[i] = act_fast_tanh(in[i]);
      break;
    case KACT_RELU:
      for (int i = 0; i < n; i++)
        out[i] = in[i] > 0.0f ? in[i] : 0.0f;
      break;
    case KACT_LEAKYRELU:
      for (int i = 0; i < n; i++)
        out[i] = in[i] > 0.0f ? in[i] : A.p0 * in[i];
      break;
    case KACT_SIGMOID:
      for (int i = 0; i < n; i++)
        out[i] = act_sigmoid(in[i]);
      break;
    default: // the rarer ones share the scalar implementation
      for (int i = 0; i < n; i++)
        out[i] = g_act1(c, A, in[i], i);
      break;
  }
}

// y[o .. o+3] (= 0 | += ) W_tap x, four outputs at a time (weights [in][out_pad], one float4 per input: the four FMA
// chains of a group are independent, one weight load feeds four of them); the bias, when given, is added once the sum
// is complete -- the reference's order (conv1d.cpp:769, dsp.cpp:832-834).  The models that reach this kernel are narrow
// (wavenet_a2_max.nam: 3..8 wide), so the input loop is kept rolled: an unrolled-by-8 loop with its remainder
// handling cost more instructions than the arithmetic.
// (Taking this and the other helpers out of line shrinks the kernel several times over, but was slower: the calls and
// the generic-address loads of the local vectors cost more than the instruction fetches they save.)
__device__ __forceinline__ void g_accumulate(const float* __restrict__ wt, const int in, const int op, const float* x,
                                             float* y, const bool from_zero, const float* __restrict__ bias)
{
  for (int o = 0; o < op; o += 4)
  {
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
    if (!from_zero)
      a0 = y[o], a1 = y[o + 1], a2 = y[o + 2], a3 = y[o + 3];
    const float4* __restrict__ w4 = reinterpret_cast<const float4*>(wt + o);
    const int stride4 = op >> 2;
    if ((in & 7) == 0)
    {
#pragma unroll 8
      for (int i = 0; i < in; i++)
      {
        const float4 w = w4[(size_t)i * stride4];
        const float xi = x[i];
        a0 = fmaf(w.x, xi, a0), a1 = fmaf(w.y, xi, a1), a2 = fmaf(w.z, xi, a2), a3 = fmaf(w.w, xi, a3);
      }
    }
    else
    {
#pragma unroll 1
      for (int i = 0; i < in; i++)
      {
        const float4 w = w4[(size_t)i * stride4];
        const float xi = x[i];
        a0 = fmaf(w.x, xi, a0), a1 = fmaf(w.y, xi, a1), a2 = fmaf(w.z, xi, a2), a3 = fmaf(w.w, xi, a3);
      }
    }
    if (bias != nullptr)
    {
      const float4 b = *reinterpret_cast<const float4*>(bias + o);
      a0 += b.x, a1 += b.y, a2 += b.z, a3 += b.w;
    }
    y[o] = a0, y[o + 1] = a1, y[o + 2] = a2, y[o + 3] = a3;
  }
}

// y = W x (+ b).  y is written up to out rounded up to 4 (the padding rows are zero): every caller's buffer has room.
__device__ __forceinline__ void g_matvec(const GenThread& c, const GMat& M, const float* x, float* y)
{
  g_accumulate(c.w + M.w_off, M.in, (M.out + 3) & ~3, x, y, true, M.b_off >= 0 ? c.w + M.b_off : nullptr);
}

// causal dilated convolution over the tile: every thread persists its x[t] in the ring, then reads x[t - off]
// (earlier threads' columns of this tile, or earlier calls'; zeros before the reset).  Called by all threads of the
// CTA in step (the control flow depends on the descriptors only).  Sums run taps oldest -> newest, inputs ascending.
__device__ __forceinline__ void g_conv(const GenThread& c, const GConv& V, const float* x, float* y)
{
  const int K = V.kernel;
  if (K > 1)
  {
    if (c.valid)
    {
      float* __restrict__ dst = c.st + V.ring_off + (long)(c.t & (uint32_t)V.ring_mask) * V.in;
      for (int i = 0; i < V.in; i++)
        dst[i] = x[i];
    }
    __syncthreads();
  }
  const int op = (V.out + 3) & ~3;
  float tap[kGenMaxVec];
  for (int k = 0; k < K; k++)
  {
    const int off = (K - 1 - k) * V.dilation;
    const float* src = x;
    if (off != 0)
    {
      const float* __restrict__ rs = c.st + V.ring_off + (long)((c.t - (uint32_t)off) & (uint32_t)V.ring_mask) * V.in;
      for (int i = 0; i < V.in; i++)
        tap[i] = __ldcg(rs + i);
      src = tap;
    }
    g_accumulate(c.w + V.w_off + (long)k * V.in * op, V.in, op, src, y, k == 0,
                 (k + 1 == K && V.b_off >= 0) ? c.w + V.b_off : nullptr);
  }
  if (K > 1)
    __syncthreads(); // every tap of this tile is read before the next tile's columns land in the ring
}

// FiLM (film.h:76-190): out = in * scale(cond) (+ shift(cond)); in place is allowed (out == in)
__device__ __forceinline__ void g_film(const GenThread& c, const GFilm& F, const float* in, const float* cond, float* out)
{
  float ss[2 * kGenMaxVec];
  g_matvec(c, F.css, cond, ss);
  if (F.shift)
    for (int i = 0; i < F.dim; i++)
      out[i] = in[i] * ss[i] + ss[F.dim + i];
  else
    for (int i = 0; i < F.dim; i++)
      out[i] = in[i] * ss[i];
}

// Layer::Process for one frame (model.cpp:183-393): x (channels) -> x_next (channels), head contribution
// (head_out_size) added to head_acc
__device__ __forceinline__ void g_layer(const GenThread& c, const GLayer& L, float* x, const float* cond, float* head_acc)
{
  const int C = L.channels, Bn = L.bottleneck, Z = L.zrows;
  float z[2 * kGenMaxVec], u[2 * kGenMaxVec];
  // input convolution with optional pre / post FiLM (:189-204)
  if (L.film[0].active)
  {
    g_film(c, L.film[0], x, cond, u);
    g_conv(c, L.conv, u, z);
  }
  else
    g_conv(c, L.conv, x, z);
  if (L.film[1].active)
    g_film(c, L.film[1], z, cond, z);
  // input mixin (:206-219)
  if (L.film[2].active)
  {
    float cf[kGenMaxVec];
    g_film(c, L.film[2], cond, cond, cf);
    g_matvec(c, L.mixin, cf, u);
  }
  else
    g_matvec(c, L.mixin, cond, u);
  if (L.film[3].active)
    g_film(c, L.film[3], u, cond, u);
  for (int i = 0; i < Z; i++)
    z[i] += u[i]; // :220-221
  if (L.film[4].active)
    g_film(c, L.film[4], z, cond, z);

  // activation (:234-288); the activated block is the first `bottleneck` entries of z
  if (L.gating == 0)
    g_act_vec(c, L.act, z, z, Z);
  else
  {
    // (u is free here: the mixin sum has been added to z)
    g_act_vec(c, L.act, z, u, Bn);
    g_act_vec(c, L.sec, z + Bn, u + Bn, Bn);
    if (L.gating == 1)
      for (int i = 0; i < Bn; i++)
        z[i] = u[i] * u[Bn + i]; // gating_activations.h:100-113
    else
      for (int i = 0; i < Bn; i++)
        z[i] = u[Bn + i] * u[i] + (1.0f - u[Bn + i]) * z[i]; // :209-227
  }
  if (L.film[5].active)
    g_film(c, L.film[5], z, cond, z);
  // head output (:290-352)
  if (L.has_h1x1)
  {
    g_matvec(c, L.h1x1, z, u);
    if (L.film[7].active)
      g_film(c, L.film[7], u, cond, u);
    for (int i = 0; i < L.h1x1.out; i++)
      head_acc[i] += u[i];
  }
  else
    for (int i = 0; i < Bn; i++)
      head_acc[i] += z[i];
  // layer1x1 + residual (:243,279-287,354-392); reference quirk: layer1x1_post_film is applied only in
  // BLENDED mode
  if (L.has_l1x1)
  {
    g_matvec(c, L.l1x1, z, u);
    if (L.gating == 2 && L.film[6].active)
      g_film(c, L.film[6], u, cond, u);
    for (int i = 0; i < C; i++)
      x[i] += u[i];
  }
}

// one frame through a whole network: in (in_channels), cond (its condition vector) -> out (out_channels)
// (head_scale: N.head_scale, or in a bank the stream's model's, from its blob)
__device__ __forceinline__ void g_net(const GenThread& c, const GNet& N, const GLayer* __restrict__ layers,
                                      const float* in, const float* cond, float* out, const float head_scale)
{
  float x[kGenMaxVec], xin[kGenMaxVec], head[kGenMaxVec], hout[kGenMaxVec];
  for (int i = 0; i < N.in_channels; i++)
    xin[i] = in[i];
  for (int a = 0; a < N.n_arrays; a++)
  {
    const GArray& A = N.arrays[a];
    // head accumulator: zeros for the first array, the previous array's head output after (model.cpp:469-486)
    for (int i = 0; i < A.head_out_size; i++)
      head[i] = (a == 0) ? 0.0f : hout[i];
    g_matvec(c, A.rechannel, xin, x);
    for (int l = 0; l < A.n_layers; l++)
      g_layer(c, layers[A.layer0 + l], x, cond, head);
    g_conv(c, A.head, head, hout);
    for (int i = 0; i < A.channels; i++)
      xin[i] = x[i];
  }
  const GArray& last = N.arrays[N.n_arrays - 1];
  if (N.with_head)
  {
    // post-stack head (model.cpp:854-883, Head::process :87-103): repeated activation -> Conv1D
    float cur[kGenMaxVec], nxt[kGenMaxVec];
    for (int i = 0; i < last.head_size; i++)
      cur[i] = head_scale * hout[i];
    for (int h = 0; h < N.n_head_convs; h++)
    {
      const GConv& V = N.head_convs[h];
      for (int i = 0; i < V.in; i++)
        cur[i] = g_act1(c, N.head_act, cur[i], i);
      g_conv(c, V, cur, nxt);
      for (int i = 0; i < V.out; i++)
        cur[i] = nxt[i];
    }
    for (int i = 0; i < N.out_channels; i++)
      out[i] = cur[i];
  }
  else
    for (int i = 0; i < N.out_channels; i++)
      out[i] = head_scale * hout[i];
}

// Model banks (BANK; a bank's calls always carry a table): position s runs the blob of model slots[s].model, at
// weights + model * weight_stride.  With WS the CTA keeps the blob of the model it staged last and restages only when the
// next position's model differs (the condition is uniform over the CTA, so the barriers around the copy are too).
template <bool WS, bool BANK, typename P>
__device__ __forceinline__ void g_bank_select(GenThread& c, const P& p, const int s, int& staged)
{
  if constexpr (BANK)
  {
    const int model = p.slots[s].model;
    const float* __restrict__ blob = p.weights + (size_t)model * p.weight_stride;
    if constexpr (WS)
    {
      if (model != staged)
      {
        __syncthreads(); // every thread is done with the previous model's weights
        extern __shared__ float4 gen_smem4[];
        const float4* src = reinterpret_cast<const float4*>(blob);
        for (int i = threadIdx.x; i < p.n_weight_floats / 4; i += kGenTile)
          gen_smem4[i] = __ldg(src + i);
        __syncthreads();
        staged = model;
      }
    }
    else
      c.w = blob;
  }
}

// The C ABI's batched entry; persistent CTAs, one stream at a time.  Multi-channel models (model.cpp:809-820,
// :888-909): stream s's channel c is the plane in[s * in_stride + c * n_frames ..] (out likewise); the input vector
// is both the first array's layer input and -- unless a condition_dsp produces it -- the condition.
// TBL: the call carries a slot table (its own instantiation: a call without one runs the table-free code).
// WS: the weight blob is staged in shared memory once per CTA (it fits for every model the kernel accepts in
// practice: example_models/wavenet_a2_max.nam is 7.5 KB); otherwise it is read through the read-only path.
template <bool WS, bool TBL = false, bool BANK = false>
__global__ void __launch_bounds__(kGenTile) wavenet_generic_kernel(const __grid_constant__ GenericKernelParams p)
{
  static_assert(TBL || !BANK, "a bank's calls carry a slot table");
  extern __shared__ float4 gen_smem4[];
  GenThread c;
  c.w = p.weights;
  int staged = -1; // BANK && WS: the model whose blob is in shared memory
  if constexpr (BANK && WS)
    c.w = reinterpret_cast<const float*>(gen_smem4);
  if constexpr (WS && !BANK)
  {
    const float4* src = reinterpret_cast<const float4*>(p.weights);
    for (int i = threadIdx.x; i < p.n_weight_floats / 4; i += kGenTile)
      gen_smem4[i] = __ldg(src + i);
    __syncthreads();
    c.w = reinterpret_cast<const float*>(gen_smem4);
  }
  const int ci = p.net.in_channels, co = p.net.out_channels;
  for (int s = blockIdx.x; s < p.batch; s += gridDim.x)
  {
    // position s of the call: state row, clock and frame count from the slot table, or row s at the handle's clock
    // (p.n_frames stays the channel-plane pitch)
    const uint32_t clock = TBL ? p.slots[s].clock : p.t_base;
    const int n = TBL ? p.slots[s].frames : p.n_frames;
    c.st = p.state + (size_t)(TBL ? p.slots[s].stream : s) * p.state_stride;
    const float* __restrict__ xin = p.in + (size_t)s * p.in_stride;
    float* __restrict__ yout = p.out + (size_t)s * p.out_stride;
    g_bank_select<WS, BANK>(c, p, s, staged);
    float bank_scale[2] = {0.0f, 0.0f}; // BANK: the position's model's output scales (net, cond), read once per position
    if constexpr (BANK)
      bank_scale[0] = c.w[p.scale_off], bank_scale[1] = c.w[p.scale_off + 1];
    for (int t0 = 0; t0 < n; t0 += kGenTile)
    {
      const int f = t0 + (int)threadIdx.x;
      c.valid = f < n;
      c.t = clock + (uint32_t)f;
      float in[kGenMaxVec], out[kGenMaxVec], cond[kGenMaxVec];
      for (int ch = 0; ch < ci; ch++)
        in[ch] = c.valid ? __ldg(xin + (size_t)ch * p.n_frames + f) : 0.0f;
      if (p.has_cond)
        g_net(c, p.cond, p.layers, in, in, cond, BANK ? bank_scale[1] : p.cond.head_scale); // _process_condition (model.cpp:777-807)
      else
        for (int ch = 0; ch < ci; ch++)
          cond[ch] = in[ch];
      g_net(c, p.net, p.layers, in, cond, out, BANK ? bank_scale[0] : p.net.head_scale);
      if (c.valid)
        for (int ch = 0; ch < co; ch++)
          yout[(size_t)ch * p.n_frames + f] = out[ch];
    }
  }
}

// ConvNet (NAM/convnet.cpp:204-272): the same frame-per-thread tiling; a block is Conv1D(kernel 2, dilation d) ->
// BatchNorm as two separate roundings, multiply then add (convnet.cpp:39-46) -> activation (:66-88); head W x + b.
// BANK: as wavenet_generic_kernel's (a ConvNet has no output scale).
template <bool WS, bool TBL = false, bool BANK = false>
__global__ void __launch_bounds__(kGenTile) convnet_kernel(const __grid_constant__ ConvNetKernelParams p)
{
  static_assert(TBL || !BANK, "a bank's calls carry a slot table");
  extern __shared__ float4 gen_smem4[];
  GenThread c;
  c.w = p.weights;
  int staged = -1;
  if constexpr (BANK && WS)
    c.w = reinterpret_cast<const float*>(gen_smem4);
  if constexpr (WS && !BANK)
  {
    const float4* src = reinterpret_cast<const float4*>(p.weights);
    for (int i = threadIdx.x; i < p.n_weight_floats / 4; i += kGenTile)
      gen_smem4[i] = __ldg(src + i);
    __syncthreads();
    c.w = reinterpret_cast<const float*>(gen_smem4);
  }
  const GConvNet& N = p.net;
  for (int s = blockIdx.x; s < p.batch; s += gridDim.x)
  {
    const uint32_t clock = TBL ? p.slots[s].clock : p.t_base;
    const int n = TBL ? p.slots[s].frames : p.n_frames;
    c.st = p.state + (size_t)(TBL ? p.slots[s].stream : s) * p.state_stride;
    const float* __restrict__ xin = p.in + (size_t)s * p.in_stride;
    float* __restrict__ yout = p.out + (size_t)s * p.out_stride;
    g_bank_select<WS, BANK>(c, p, s, staged);
    for (int t0 = 0; t0 < n; t0 += kGenTile)
    {
      const int f = t0 + (int)threadIdx.x;
      c.valid = f < n;
      c.t = clock + (uint32_t)f;
      float x[kGenMaxVec], z[kGenMaxVec];
      for (int ch = 0; ch < N.in_channels; ch++)
        x[ch] = c.valid ? __ldg(xin + (size_t)ch * p.n_frames + f) : 0.0f;
      for (int b = 0; b < N.n_blocks; b++)
      {
        g_conv(c, N.convs[b], x, z);
        if (N.bn_off[b] >= 0)
        {
          const float* __restrict__ sc = c.w + N.bn_off[b];
          for (int j = 0; j < N.channels; j++)
            z[j] = __fadd_rn(__fmul_rn(z[j], sc[j]), sc[N.channels + j]);
        }
        g_act_vec(c, N.act, z, x, N.channels);
      }
      g_matvec(c, N.head, x, z);
      if (c.valid)
        for (int ch = 0; ch < N.out_channels; ch++)
          yout[(size_t)ch * p.n_frames + f] = z[ch];
    }
  }
}

} // namespace namb200
