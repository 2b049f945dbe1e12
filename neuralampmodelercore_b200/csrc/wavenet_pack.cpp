#include "wavenet_pack.h"

#include <algorithm>
#include <cstdint>
#include <cstring>

namespace namb200
{

namespace
{
int pad_channels(int c)
{
  if (c <= 4)
    return 4;
  if (c <= 8)
    return 8;
  if (c <= 16)
    return 16;
  return -1;
}

int next_pow2(long v)
{
  int r = 1;
  while (r < v)
    r <<= 1;
  return r;
}

size_t align4(size_t n)
{
  return (n + 3) & ~(size_t)3;
}
} // namespace

WaveNetPlan plan_wavenet(const ModelSpec& ms)
{
  WaveNetPlan plan;
  const WaveNetSpec& wn = ms.wavenet;
  auto no = [&plan](const std::string& why) {
    plan.eligible = false;
    plan.why_not = why;
    return plan;
  };
  if (ms.arch != Arch::WaveNet)
    return no("not a WaveNet");
  if (wn.in_channels != 1 || ms.out_channels != 1)
    return no("fused kernel is mono in / mono out (in_channels " + std::to_string(wn.in_channels) + ", out_channels "
              + std::to_string(ms.out_channels) + ")");
  if (wn.condition_dsp)
    return no("condition_dsp sub-model");
  if (wn.with_head)
    return no("post-stack head");
  if (wn.arrays.empty() || wn.arrays.size() > 2)
    return no(std::to_string(wn.arrays.size()) + " layer arrays (fused kernel handles 1 or 2)");
  plan.n_arrays = (int)wn.arrays.size();
  size_t total_layers = 0;
  for (size_t a = 0; a < wn.arrays.size(); a++)
  {
    const ArraySpec& A = wn.arrays[a];
    const std::string where = "layer array " + std::to_string(a) + ": ";
    if (A.condition_size != 1)
      return no(where + "condition_size " + std::to_string(A.condition_size));
    if (A.bottleneck != A.channels)
      return no(where + "bottleneck != channels");
    if (pad_channels(A.channels) < 0)
      return no(where + std::to_string(A.channels) + " channels (max 16)");
    if (A.groups_input != 1 || A.groups_input_mixin != 1 || A.l1x1_groups != 1)
      return no(where + "grouped convolutions");
    if (!A.l1x1_active)
      return no(where + "layer1x1 inactive");
    if (A.h1x1_active)
      return no(where + "head1x1");
    if ((A.head_kernel - 1) * A.head_dilation > kHalo)
      return no(where + "head convolution looks back " + std::to_string((A.head_kernel - 1) * A.head_dilation)
                + " frames (max " + std::to_string(kHalo) + ")");
    const int expect_in = (a == 0) ? 1 : wn.arrays[a - 1].channels;
    if (A.input_size != expect_in)
      return no(where + "input_size " + std::to_string(A.input_size) + " (expected " + std::to_string(expect_in) + ")");
    for (const LayerSpec& L : A.layers)
    {
      if (L.gating != Gating::None)
        return no(where + "gated / blended activation");
      for (int f = 0; f < F_COUNT; f++)
        if (L.film[f].active)
          return no(where + "FiLM");
      if (L.act.type == ActType::PReLU && L.act.slopes.size() != 1 && (int)L.act.slopes.size() != A.channels)
        return no(where + "PReLU slope count");
    }
    total_layers += A.layers.size();
    plan.cp[a] = pad_channels(A.channels);
    plan.creal[a] = A.channels;
  }
  if (wn.arrays.back().head_size != 1)
    return no("last head_size != 1");
  if (total_layers > (size_t)kMaxLayers)
    return no("too many layers");

  // ---- pack ----
  std::vector<float>& blob = plan.blob;
  long ring_off = 0;
  double macs = 0.0;
  for (size_t a = 0; a < wn.arrays.size(); a++)
  {
    const ArraySpec& A = wn.arrays[a];
    const int C = plan.cp[a], Cr = A.channels;
    const int CIN = (a == 0) ? 1 : plan.cp[a - 1];
    const int CINr = A.input_size;
    const bool is_last = (a + 1 == wn.arrays.size());
    const int HOUT = is_last ? 1 : plan.cp[a + 1];
    const int HOUTr = A.head_size;
    ArrayDesc ad;
    ad.layer0 = (int)plan.layers.size();
    ad.n_layers = (int)A.layers.size();
    // rechannel [CIN][C]
    ad.rech_off = (int)blob.size();
    blob.resize(blob.size() + (size_t)CIN * C, 0.0f);
    for (int i = 0; i < CINr; i++)
      for (int o = 0; o < Cr; o++)
        blob[ad.rech_off + (size_t)i * C + o] = A.rechannel.w[(size_t)o * CINr + i];
    macs += (double)CINr * Cr;
    for (const LayerSpec& L : A.layers)
    {
      LayerDesc ld{};
      const int K = L.conv.kernel;
      ld.w_off = (int)blob.size();
      ld.kernel = K;
      ld.dilation = L.conv.dilation;
      ld.lookback = (int)L.conv.lookback();
      if (ld.lookback > plan.max_lookback)
        plan.max_lookback = ld.lookback;
      const int R = next_pow2(ld.lookback > 0 ? ld.lookback : 1);
      ld.ring_mask = R - 1;
      ld.ring_off = (int)ring_off;
      ring_off += (long)C * R;
      ld.act = (int)L.act.type;
      ld.ap0 = ld.ap1 = ld.ap2 = ld.ap3 = 0.0f;
      if (L.act.type == ActType::LeakyReLU)
        ld.ap0 = L.act.slope;
      else if (L.act.type == ActType::LeakyHardtanh)
      {
        ld.ap0 = L.act.min_val;
        ld.ap1 = L.act.max_val;
        ld.ap2 = L.act.min_slope;
        ld.ap3 = L.act.max_slope;
      }
      // conv [K][C(in)][C(out)]
      const size_t conv_off = blob.size();
      blob.resize(blob.size() + (size_t)K * C * C, 0.0f);
      for (int k = 0; k < K; k++)
        for (int i = 0; i < Cr; i++)
          for (int o = 0; o < Cr; o++)
            blob[conv_off + ((size_t)k * C + i) * C + o] = L.conv.w[((size_t)k * Cr + o) * Cr + i];
      // bias [C]
      const size_t b_off = blob.size();
      blob.resize(blob.size() + C, 0.0f);
      for (int o = 0; o < Cr; o++)
        blob[b_off + o] = L.conv.b[o];
      // mixin [C]  (condition_size == 1)
      const size_t m_off = blob.size();
      blob.resize(blob.size() + C, 0.0f);
      for (int o = 0; o < Cr; o++)
        blob[m_off + o] = L.mixin.w[o];
      // layer1x1 P [C(in)][C(out)], bias [C]
      const size_t p_off = blob.size();
      blob.resize(blob.size() + (size_t)C * C, 0.0f);
      for (int i = 0; i < Cr; i++)
        for (int o = 0; o < Cr; o++)
          blob[p_off + (size_t)i * C + o] = L.l1x1.w[(size_t)o * Cr + i];
      const size_t pb_off = blob.size();
      blob.resize(blob.size() + C, 0.0f);
      for (int o = 0; o < Cr; o++)
        blob[pb_off + o] = L.l1x1.b[o];
      // PReLU slopes [C]
      const size_t s_off = blob.size();
      blob.resize(blob.size() + C, 0.0f);
      if (L.act.type == ActType::PReLU)
        for (int o = 0; o < Cr; o++)
          blob[s_off + o] = L.act.slopes.size() == 1 ? L.act.slopes[0] : L.act.slopes[o];
      macs += (double)K * Cr * Cr + Cr + (double)Cr * Cr;
      plan.layers.push_back(ld);
    }
    // head rechannel [HK][C(in)][HOUT] + bias[HOUT], padded to a multiple of 4 floats
    const int HK = A.head_kernel;
    ad.head_kernel = HK;
    ad.head_dilation = A.head_dilation;
    ad.head_off = (int)blob.size();
    blob.resize(blob.size() + align4((size_t)HK * C * HOUT + HOUT), 0.0f);
    for (int k = 0; k < HK; k++)
      for (int i = 0; i < Cr; i++)
        for (int o = 0; o < HOUTr; o++)
          blob[ad.head_off + ((size_t)k * C + i) * HOUT + o] = A.head_rechannel.w[((size_t)k * HOUTr + o) * Cr + i];
    if (A.head_rechannel.bias)
      for (int o = 0; o < HOUTr; o++)
        blob[ad.head_off + (size_t)HK * C * HOUT + o] = A.head_rechannel.b[o];
    macs += (double)HK * Cr * HOUTr;
    ad.head_ring_off = 0;
    ad.head_ring_mask = 0;
    if (HK > 1)
    {
      const int hl = (HK - 1) * A.head_dilation;
      const int R = next_pow2(hl);
      ad.head_ring_off = (int)ring_off;
      ad.head_ring_mask = R - 1;
      ring_off += (long)C * R;
      if (hl > plan.max_lookback)
        plan.max_lookback = hl;
    }
    plan.arrays.push_back(ad);
  }
  blob.resize(align4(blob.size()), 0.0f);
  plan.state_floats = (ring_off + 31) & ~31L;
  plan.head_scale = wn.head_scale;
  plan.macs_per_frame = macs;
  plan.eligible = true;
  return plan;
}

} // namespace namb200
