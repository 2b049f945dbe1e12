#include "generic_pack.h"

#include <algorithm>

namespace namb200
{

namespace
{

struct Packer
{
  GenericPlan& plan;
  std::string err;

  int put(const std::vector<float>& v)
  {
    const int off = (int)plan.weights.size();
    plan.weights.insert(plan.weights.end(), v.begin(), v.end());
    return off;
  }
  // 16-byte aligned, padded with zeros to a multiple of 4 floats (the kernel reads float4s)
  int put4(const std::vector<float>& v)
  {
    plan.weights.resize((plan.weights.size() + 3) & ~(size_t)3, 0.0f);
    const int off = (int)plan.weights.size();
    plan.weights.insert(plan.weights.end(), v.begin(), v.end());
    plan.weights.resize((plan.weights.size() + 3) & ~(size_t)3, 0.0f);
    return off;
  }
  // `taps` (out x in) row-major matrices -> [tap][in][out_pad], out_pad = out rounded up to 4: one float4 holds the
  // weights of four outputs for one input, the layout the kernel's 4-output accumulation wants
  int put_transposed(const std::vector<float>& w, int taps, int in, int out)
  {
    const int op = (out + 3) & ~3;
    std::vector<float> t((size_t)taps * in * op, 0.0f);
    for (int k = 0; k < taps; k++)
      for (int o = 0; o < out; o++)
        for (int i = 0; i < in; i++)
          t[((size_t)k * in + i) * op + o] = w[((size_t)k * out + o) * in + i];
    return put4(t);
  }
  bool width(int n, const char* what)
  {
    if (n < 1 || n > kGenMaxVec)
    {
      if (err.empty())
        err = std::string(what) + " " + std::to_string(n) + " (general kernel handles 1.." + std::to_string(kGenMaxVec) + ")";
      return false;
    }
    return true;
  }
  GMat mat(const Conv1x1W& m)
  {
    GMat g{};
    g.in = m.in;
    g.out = m.out;
    width(m.in, "matrix input width");
    width(m.out, "matrix output width");
    if ((long)m.w.size() != (long)m.in * m.out)
    {
      if (err.empty())
        err = "internal: 1x1 weight count";
      return g;
    }
    g.w_off = put_transposed(m.w, 1, m.in, m.out);
    g.b_off = m.bias ? put4(m.b) : -1;
    plan.macs_per_frame += (double)m.in * m.out / std::max(m.groups, 1);
    return g;
  }
  GConv conv(const Conv1DW& v)
  {
    GConv g{};
    g.in = v.in;
    g.out = v.out;
    g.kernel = v.kernel;
    g.dilation = v.dilation;
    width(v.in, "convolution input width");
    width(v.out, "convolution output width");
    if ((long)v.w.size() != (long)v.kernel * v.in * v.out)
    {
      if (err.empty())
        err = "internal: conv weight count";
      return g;
    }
    g.w_off = put_transposed(v.w, v.kernel, v.in, v.out);
    g.b_off = v.bias ? put4(v.b) : -1;
    g.ring_mask = 0;
    g.ring_off = (int)plan.state_floats;
    if (v.kernel > 1)
    {
      long r = 1;
      while (r < v.lookback() + kGenTile)
        r <<= 1;
      g.ring_mask = (int)(r - 1);
      plan.state_floats += r * v.in;
    }
    plan.macs_per_frame += (double)v.kernel * v.in * v.out / std::max(v.groups, 1);
    return g;
  }
  GAct act(const ActSpec& a)
  {
    GAct g{};
    g.type = (int)a.type;
    g.slopes_off = 0;
    g.n_slopes = 0;
    if (a.type == ActType::LeakyReLU)
      g.p0 = a.slope;
    else if (a.type == ActType::LeakyHardtanh)
    {
      g.p0 = a.min_val;
      g.p1 = a.max_val;
      g.p2 = a.min_slope;
      g.p3 = a.max_slope;
    }
    else if (a.type == ActType::PReLU)
    {
      g.slopes_off = put(a.slopes);
      g.n_slopes = (int)a.slopes.size();
      if (a.slopes.empty() && err.empty())
        err = "PReLU without slopes";
    }
    return g;
  }
  GFilm film(const FilmSpec& f)
  {
    GFilm g{};
    g.active = f.active ? 1 : 0;
    if (!f.active)
      return g;
    g.shift = f.shift ? 1 : 0;
    g.dim = f.dim;
    width(f.dim, "FiLM width");
    g.css = mat(f.css);
    plan.macs_per_frame += f.dim;
    return g;
  }

  bool net(const WaveNetSpec& wn, int out_channels, GNet& N)
  {
    N = GNet{};
    N.in_channels = wn.in_channels;
    N.out_channels = out_channels;
    N.head_scale = wn.head_scale;
    if (wn.arrays.empty() || (int)wn.arrays.size() > kGenMaxArrays)
    {
      err = std::to_string(wn.arrays.size()) + " layer arrays (general kernel handles 1.." + std::to_string(kGenMaxArrays) + ")";
      return false;
    }
    N.n_arrays = (int)wn.arrays.size();
    for (size_t a = 0; a < wn.arrays.size(); a++)
    {
      const ArraySpec& A = wn.arrays[a];
      GArray& G = N.arrays[a];
      G.input_size = A.input_size;
      G.channels = A.channels;
      G.head_out_size = A.head_out_size();
      G.head_size = A.head_size;
      G.layer0 = (int)plan.layers.size();
      G.n_layers = (int)A.layers.size();
      // the config's widths, named as the config names them (the matrices below would only say "matrix output width")
      width(A.channels, "channels");
      width(A.condition_size, "condition size");
      width(A.head_size, "head size");
      for (const LayerSpec& L : A.layers)
      {
        width(L.conv.out, L.gating == Gating::None ? "bottleneck" : "2 x bottleneck (gated / blended layer)");
        if (L.has_h1x1)
          width(L.h1x1.out, "head1x1 out_channels");
      }
      if (a > 0 && wn.arrays[a - 1].head_size != A.head_out_size() && err.empty())
        err = "head size of array " + std::to_string(a - 1) + " does not feed array " + std::to_string(a);
      G.rechannel = mat(A.rechannel);
      for (const LayerSpec& L : A.layers)
      {
        GLayer g{};
        g.channels = A.channels;
        g.bottleneck = A.bottleneck;
        g.gating = (int)L.gating;
        g.zrows = L.conv.out;
        g.has_l1x1 = L.has_l1x1 ? 1 : 0;
        g.has_h1x1 = L.has_h1x1 ? 1 : 0;
        g.conv = conv(L.conv);
        g.mixin = mat(L.mixin);
        if (L.has_l1x1)
          g.l1x1 = mat(L.l1x1);
        if (L.has_h1x1)
          g.h1x1 = mat(L.h1x1);
        g.act = act(L.act);
        g.sec = act(L.sec_act);
        for (int f = 0; f < kGenFilmSites; f++)
          g.film[f] = film(L.film[f]);
        plan.layers.push_back(g);
      }
      G.head = conv(A.head_rechannel);
    }
    N.with_head = wn.with_head ? 1 : 0;
    if (wn.with_head)
    {
      if ((int)wn.post_head.convs.size() > kGenMaxHeadConvs)
      {
        err = "post-stack head with " + std::to_string(wn.post_head.convs.size()) + " convolutions (general kernel handles up to "
              + std::to_string(kGenMaxHeadConvs) + ")";
        return false;
      }
      N.n_head_convs = (int)wn.post_head.convs.size();
      N.head_act = act(wn.post_head.act);
      for (size_t i = 0; i < wn.post_head.convs.size(); i++)
        N.head_convs[i] = conv(wn.post_head.convs[i]);
    }
    return err.empty();
  }
};

} // namespace

GenericPlan plan_generic(const ModelSpec& ms)
{
  GenericPlan plan;
  auto no = [&plan](const std::string& why) {
    plan.eligible = false;
    plan.why_not = why;
    return plan;
  };
  if (ms.arch != Arch::WaveNet)
    return no("not a WaveNet");
  const WaveNetSpec& wn = ms.wavenet;
  Packer pk{plan, {}};
  if (!pk.width(wn.in_channels, "input channels") || !pk.width(ms.out_channels, "output channels"))
    return no(pk.err);
  if (!pk.net(wn, ms.out_channels, plan.net))
    return no(pk.err);
  if (wn.condition_dsp)
  {
    const ModelSpec& cm = *wn.condition_dsp;
    if (cm.arch != Arch::WaveNet)
      return no("condition_dsp is not a WaveNet");
    if (cm.wavenet.condition_dsp)
      return no("nested condition_dsp");
    if (cm.wavenet.in_channels != wn.in_channels) // model.cpp:603-611
      return no("input channels of WaveNet (" + std::to_string(wn.in_channels)
                + ") don't match input channels of condition DSP (" + std::to_string(cm.wavenet.in_channels) + ")");
    if (!pk.net(cm.wavenet, cm.out_channels, plan.cond))
      return no("condition_dsp: " + pk.err);
    if (!pk.width(cm.out_channels, "condition_dsp output width"))
      return no(pk.err);
    plan.has_cond = true;
  }
  // the input vector is the first array's layer input and, without a condition_dsp, every array's condition
  // (model.cpp:809-820,840; the reference leaves a mismatch to an Eigen assertion)
  if (wn.arrays[0].input_size != wn.in_channels)
    return no("input_size of the first layer array (" + std::to_string(wn.arrays[0].input_size) + ") != in_channels ("
              + std::to_string(wn.in_channels) + ")");
  const int cond_dim = plan.has_cond ? wn.condition_dsp->out_channels : wn.in_channels;
  for (const ArraySpec& A : wn.arrays)
    if (A.condition_size != cond_dim)
      return no("condition_size " + std::to_string(A.condition_size) + " != condition width " + std::to_string(cond_dim));
  if (!pk.err.empty())
    return no(pk.err);
  plan.weights.resize((plan.weights.size() + 3) & ~(size_t)3, 0.0f);
  plan.state_floats = (plan.state_floats + 3) & ~3L;
  plan.eligible = true;
  return plan;
}

GenericPlan plan_convnet(const ModelSpec& ms)
{
  GenericPlan plan;
  auto no = [&plan](const std::string& why) {
    plan.eligible = false;
    plan.why_not = why;
    return plan;
  };
  if (ms.arch != Arch::ConvNet)
    return no("not a ConvNet");
  const ConvNetSpec& cn = ms.convnet;
  if ((int)cn.blocks.size() > kGenMaxBlocks)
    return no(std::to_string(cn.blocks.size()) + " ConvNet blocks (kernel handles up to " + std::to_string(kGenMaxBlocks) + ")");
  Packer pk{plan, {}};
  GConvNet& N = plan.convnet;
  N = GConvNet{};
  N.in_channels = ms.in_channels;
  N.out_channels = ms.out_channels;
  N.channels = cn.channels;
  N.n_blocks = (int)cn.blocks.size();
  pk.width(ms.in_channels, "input channels");
  pk.width(ms.out_channels, "output channels");
  pk.width(cn.channels, "channels");
  N.act = pk.act(cn.act);
  for (size_t i = 0; i < cn.blocks.size() && pk.err.empty(); i++)
  {
    const ConvNetSpec::Block& b = cn.blocks[i];
    N.convs[i] = pk.conv(b.conv);
    N.bn_off[i] = -1;
    if (cn.batchnorm)
    {
      std::vector<float> sl(b.scale);
      sl.insert(sl.end(), b.loc.begin(), b.loc.end());
      N.bn_off[i] = pk.put4(sl);
      plan.macs_per_frame += cn.channels;
    }
  }
  N.head = pk.mat(cn.head);
  if (!pk.err.empty())
    return no(pk.err);
  plan.weights.resize((plan.weights.size() + 3) & ~(size_t)3, 0.0f);
  plan.state_floats = (plan.state_floats + 3) & ~3L;
  plan.eligible = true;
  return plan;
}

} // namespace namb200
