// wavenet_generic_spec.cuh -- the general WaveNet kernel (wavenet_generic.cuh), compiled PER MODEL by NVRTC.
//
// wavenet_generic.cuh interprets descriptors at run time: loop bounds come from memory, every per-frame vector is a local
// array indexed by loop variables (local memory), weights are fetched from shared memory: bookkeeping, not arithmetic,
// fills the issue slots.  Here the SAME algorithm, the same summation
// order and the same ring layout are compiled together with a generated header (jit_spec.cpp) that holds the model as
// constant data: `gspec::net`, `gspec::cond`, `gspec::layers[]` (the descriptors of generic_desc.h) and the weights as bit
// patterns.  Every function below is force-inlined and every loop has, after inlining, a constant trip count, so the
// compiler unrolls the whole network into straight-line code: the vectors become registers, the descriptor fields
// constants, the weights FFMA immediates, the option switches (gating, FiLM sites, head1x1, activations) disappear.
//
// Compiled for a model bank's SHAPE (gspec::bank, jit_spec.cpp), the header holds the descriptors only: gspec::w(i) reads the
// current stream's blob from shared memory, staged when the next stream's model differs, and the output scales come from
// the blob through gspec::out_scale (the ordinary header's returns the constant).
//
// What it computes (reference, under NAM/): wavenet/model.cpp:183-393 Layer::Process, :463-549 LayerArray, :777-910
// WaveNet::process with condition_dsp, :19-103 the post-stack head; film.h:76-190; gating_activations.h:100-113,209-227.
#pragma once

#ifndef NAMB200_GSPEC_HEADER_INCLUDED
#error "include the generated model header (namespace gspec) before wavenet_generic_spec.cuh"
#endif

namespace namb200_gspec
{
using namespace namb200;

enum : int
{
  ACT_TANH = 0,
  ACT_HARDTANH = 1,
  ACT_FASTTANH = 2,
  ACT_RELU = 3,
  ACT_LEAKYRELU = 4,
  ACT_PRELU = 5,
  ACT_SIGMOID = 6,
  ACT_SILU = 7,
  ACT_HARDSWISH = 8,
  ACT_LEAKYHARDTANH = 9,
  ACT_SOFTSIGN = 10
};

constexpr int kTile = 128; // frames per tile == threads per CTA (the ring geometry of generic_pack.cpp assumes it)

struct Th
{
  float* st; // this CTA's stream
  unsigned t; // absolute index of this thread's frame
  bool valid;
};

__device__ __forceinline__ float rcp_approx(float x)
{
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float fast_tanh(float x) // activations.h:91-98
{
  const float ax = fabsf(x);
  const float x2 = x * x;
  const float num = x * (2.45550750702956f + 2.45550750702956f * ax + (0.893229853513558f + 0.821226666969744f * ax) * x2);
  const float den = 2.44506634652299f + (2.44506634652299f + x2) * fabsf(x + 0.814642734961073f * x * ax);
  return num * rcp_approx(den);
}
__device__ __forceinline__ float sigmoid(float x)
{
  return rcp_approx(1.0f + expf(-x));
}

__device__ __forceinline__ float act1(const GAct A, const float x, const int ch)
{
  switch (A.type)
  {
    case ACT_TANH: return tanhf(x);
    case ACT_FASTTANH: return fast_tanh(x);
    case ACT_HARDTANH: return fminf(fmaxf(x, -1.0f), 1.0f);
    case ACT_RELU: return x > 0.0f ? x : 0.0f;
    case ACT_LEAKYRELU: return x > 0.0f ? x : A.p0 * x;
    case ACT_PRELU: return x > 0.0f ? x : gspec::w(A.slopes_off + (A.n_slopes == 1 ? 0 : ch)) * x;
    case ACT_SIGMOID: return sigmoid(x);
    case ACT_SILU: return x * sigmoid(x);
    case ACT_HARDSWISH:
    {
      const float t = x + 3.0f;
      const float cl = t < 0.0f ? 0.0f : (t > 6.0f ? 6.0f : t);
      return x * cl * (1.0f / 6.0f);
    }
    case ACT_LEAKYHARDTANH: return x < A.p0 ? (x - A.p0) * A.p2 + A.p0 : (x > A.p1 ? (x - A.p1) * A.p3 + A.p1 : x);
    case ACT_SOFTSIGN: return x * rcp_approx(1.0f + fabsf(x));
    default: return x;
  }
}
__device__ __forceinline__ void act_vec(const GAct A, const float* in, float* out, const int n)
{
#pragma unroll
  for (int i = 0; i < n; i++)
    out[i] = act1(A, in[i], i);
}

// y[0 .. op) (= 0 | +=) W_tap x; weights [in][op] at w_off; the bias, when given (b_off >= 0), is added once the sum is
// complete -- the reference's order (conv1d.cpp:769, dsp.cpp:832-834).  Same order as g_accumulate: inputs ascending.
__device__ __forceinline__ void accumulate(const int w_off, const int in, const int op, const float* x, float* y,
                                           const bool from_zero, const int b_off)
{
#pragma unroll
  for (int o = 0; o < op; o++)
  {
    float a = from_zero ? 0.0f : y[o];
#pragma unroll
    for (int i = 0; i < in; i++)
      a = fmaf(gspec::w(w_off + i * op + o), x[i], a);
    if (b_off >= 0)
      a += gspec::w(b_off + o);
    y[o] = a;
  }
}
__device__ __forceinline__ void matvec(const GMat M, const float* x, float* y)
{
  accumulate(M.w_off, M.in, (M.out + 3) & ~3, x, y, true, M.b_off);
}

// causal dilated convolution over the tile (cf. g_conv): every thread persists its x[t] in the ring, then reads x[t - off]
__device__ __forceinline__ void conv(const Th& c, const GConv V, const float* x, float* y)
{
  const int K = V.kernel;
  if (K > 1)
  {
    if (c.valid)
    {
      float* __restrict__ dst = c.st + V.ring_off + (long)(c.t & (unsigned)V.ring_mask) * V.in;
#pragma unroll
      for (int i = 0; i < V.in; i++)
        dst[i] = x[i];
    }
    __syncthreads();
  }
  const int op = (V.out + 3) & ~3;
#pragma unroll
  for (int k = 0; k < K; k++)
  {
    const int off = (K - 1 - k) * V.dilation;
    float tap[kGenMaxVec];
    if (off != 0)
    {
      const float* __restrict__ rs = c.st + V.ring_off + (long)((c.t - (unsigned)off) & (unsigned)V.ring_mask) * V.in;
#pragma unroll
      for (int i = 0; i < V.in; i++)
        tap[i] = __ldcg(rs + i);
    }
    else
    {
#pragma unroll
      for (int i = 0; i < V.in; i++)
        tap[i] = x[i];
    }
    accumulate(V.w_off + k * V.in * op, V.in, op, tap, y, k == 0, (k + 1 == K) ? V.b_off : -1);
  }
  if (K > 1)
    __syncthreads(); // every tap of this tile is read before the next tile's columns land in the ring
}

// FiLM (film.h:76-190): out = in * scale(cond) (+ shift(cond)); in place is allowed
__device__ __forceinline__ void film(const GFilm F, const float* in, const float* cond, float* out)
{
  float ss[2 * kGenMaxVec];
  matvec(F.css, cond, ss);
#pragma unroll
  for (int i = 0; i < F.dim; i++)
    out[i] = F.shift ? in[i] * ss[i] + ss[F.dim + i] : in[i] * ss[i];
}

// compile-time loops (every descriptor index must be a constant expression for the loops below to unroll)
template <int V>
struct IntC
{
  static constexpr int value = V;
};
template <int I, int N, typename F>
__device__ __forceinline__ void static_for(F&& f)
{
  if constexpr (I < N)
  {
    f(IntC<I>{});
    static_for<I + 1, N>(f);
  }
}

// Layer::Process for one frame (model.cpp:183-393), cf. g_layer
template <int LI>
__device__ __forceinline__ void layer(const Th& c, float* x, const float* cond, float* head_acc)
{
  constexpr GLayer L = gspec::layers[LI];
  constexpr int C = L.channels, Bn = L.bottleneck, Z = L.zrows;
  float z[2 * kGenMaxVec], u[2 * kGenMaxVec];
  if (L.film[0].active)
  {
    film(L.film[0], x, cond, u);
    conv(c, L.conv, u, z);
  }
  else
    conv(c, L.conv, x, z);
  if (L.film[1].active)
    film(L.film[1], z, cond, z);
  if (L.film[2].active)
  {
    float cf[kGenMaxVec];
    film(L.film[2], cond, cond, cf);
    matvec(L.mixin, cf, u);
  }
  else
    matvec(L.mixin, cond, u);
  if (L.film[3].active)
    film(L.film[3], u, cond, u);
#pragma unroll
  for (int i = 0; i < Z; i++)
    z[i] += u[i]; // :220-221
  if (L.film[4].active)
    film(L.film[4], z, cond, z);

  if (L.gating == 0)
    act_vec(L.act, z, z, Z);
  else
  {
    act_vec(L.act, z, u, Bn);
    act_vec(L.sec, z + Bn, u + Bn, Bn);
#pragma unroll
    for (int i = 0; i < Bn; i++)
      z[i] = (L.gating == 1) ? u[i] * u[Bn + i] // gating_activations.h:100-113
                             : u[Bn + i] * u[i] + (1.0f - u[Bn + i]) * z[i]; // :209-227
  }
  if (L.film[5].active)
    film(L.film[5], z, cond, z);
  if (L.has_h1x1)
  {
    matvec(L.h1x1, z, u);
    if (L.film[7].active)
      film(L.film[7], u, cond, u);
#pragma unroll
    for (int i = 0; i < L.h1x1.out; i++)
      head_acc[i] += u[i];
  }
  else
  {
#pragma unroll
    for (int i = 0; i < Bn; i++)
      head_acc[i] += z[i];
  }
  // layer1x1 + residual; reference quirk: layer1x1_post_film is applied only in BLENDED mode (model.cpp:279-287)
  if (L.has_l1x1)
  {
    matvec(L.l1x1, z, u);
    if (L.gating == 2 && L.film[6].active)
      film(L.film[6], u, cond, u);
#pragma unroll
    for (int i = 0; i < C; i++)
      x[i] += u[i];
  }
}

// one frame through a whole network (cf. g_net); COND: the condition_dsp sub-model, else the main network
template <bool COND>
__device__ __forceinline__ void net_forward(const Th& c, const float* in, const float* cond, float* out)
{
  constexpr GNet N = COND ? gspec::cond : gspec::net;
  float x[kGenMaxVec], xin[kGenMaxVec], head[kGenMaxVec], hout[kGenMaxVec];
#pragma unroll
  for (int i = 0; i < N.in_channels; i++)
    xin[i] = in[i];
  static_for<0, N.n_arrays>([&](auto a_c) {
    constexpr int a = decltype(a_c)::value;
    constexpr GArray A = N.arrays[a];
#pragma unroll
    for (int i = 0; i < A.head_out_size; i++)
      head[i] = (a == 0) ? 0.0f : hout[i];
    matvec(A.rechannel, xin, x);
    static_for<0, A.n_layers>([&](auto l_c) { layer<A.layer0 + decltype(l_c)::value>(c, x, cond, head); });
    conv(c, A.head, head, hout);
#pragma unroll
    for (int i = 0; i < A.channels; i++)
      xin[i] = x[i];
  });
  constexpr GArray last = N.arrays[N.n_arrays - 1];
  if constexpr (N.with_head != 0)
  {
    float cur[kGenMaxVec], nxt[kGenMaxVec];
#pragma unroll
    for (int i = 0; i < last.head_size; i++)
      cur[i] = gspec::out_scale(COND ? 1 : 0) * hout[i];
    static_for<0, N.n_head_convs>([&](auto h_c) {
      constexpr GConv V = N.head_convs[decltype(h_c)::value];
#pragma unroll
      for (int i = 0; i < V.in; i++)
        cur[i] = act1(N.head_act, cur[i], i);
      conv(c, V, cur, nxt);
#pragma unroll
      for (int i = 0; i < V.out; i++)
        cur[i] = nxt[i];
    });
#pragma unroll
    for (int i = 0; i < N.out_channels; i++)
      out[i] = cur[i];
  }
  else
  {
#pragma unroll
    for (int i = 0; i < N.out_channels; i++)
      out[i] = gspec::out_scale(COND ? 1 : 0) * hout[i];
  }
}

} // namespace namb200_gspec

extern "C" __global__ void __launch_bounds__(namb200_gspec::kTile) wavenet_generic_spec_kernel(const __grid_constant__ namb200::JitParams p)
{
  using namespace namb200_gspec;
  Th c;
  constexpr int ci = gspec::net.in_channels, co = gspec::net.out_channels;
  int staged = -1; // a bank's kernel: the model whose blob is in shared memory
  for (int s = blockIdx.x; s < p.batch; s += gridDim.x)
  {
    if constexpr (gspec::bank != 0)
    {
      // (a bank's calls always carry a table; the condition is uniform over the CTA, so are the barriers)
      const int model = p.slots[s].model;
      if (model != staged)
      {
        __syncthreads(); // every thread is done with the previous model's weights
        const float4* src = reinterpret_cast<const float4*>(p.weights + (size_t)model * p.weight_stride);
        for (int i = threadIdx.x; i < gspec::blob_floats / 4; i += kTile)
          gspec::blob4[i] = __ldg(src + i);
        __syncthreads();
        staged = model;
      }
    }
    const unsigned clock = p.slots ? p.slots[s].clock : p.t_base;
    const int n = p.slots ? p.slots[s].frames : p.n_frames; // (p.n_frames stays the channel-plane pitch)
    c.st = p.state + (size_t)(p.slots ? p.slots[s].stream : s) * p.state_stride;
    const float* __restrict__ xin = p.in + (size_t)s * p.in_stride;
    float* __restrict__ yout = p.out + (size_t)s * p.out_stride;
    for (int t0 = 0; t0 < n; t0 += kTile)
    {
      const int f = t0 + (int)threadIdx.x;
      c.valid = f < n;
      c.t = clock + (unsigned)f;
      float in[kGenMaxVec], out[kGenMaxVec], cond[kGenMaxVec];
#pragma unroll
      for (int ch = 0; ch < ci; ch++)
        in[ch] = c.valid ? __ldg(xin + (size_t)ch * p.n_frames + f) : 0.0f;
      if constexpr (gspec::has_cond != 0)
        net_forward<true>(c, in, in, cond); // _process_condition (model.cpp:777-807)
      else
      {
#pragma unroll
        for (int ch = 0; ch < ci; ch++)
          cond[ch] = in[ch];
      }
      net_forward<false>(c, in, cond, out);
      if (c.valid)
      {
#pragma unroll
        for (int ch = 0; ch < co; ch++)
          yout[(size_t)ch * p.n_frames + f] = out[ch];
      }
    }
  }
}
