#include "nam_model_spec.h"

#include <algorithm>
#include <cmath>
#include <cstdio>

#include <array>
#include <cctype>
#include <fstream>
#include <iostream>
#include <sstream>

namespace namb200
{

namespace
{

// ---- weight stream ---------------------------------------------------------------------------
class WeightStream
{
public:
  explicit WeightStream(const std::vector<float>& w)
  : _w(w)
  {
  }
  float next()
  {
    if (_pos >= _w.size())
    {
      // NAM/wavenet/model.cpp:681
      throw std::runtime_error("Weight mismatch: provided " + std::to_string(_w.size())
                               + " weights, but the model expects more.");
    }
    return _w[_pos++];
  }
  size_t position() const { return _pos; }
  size_t size() const { return _w.size(); }

private:
  const std::vector<float>& _w;
  size_t _pos = 0;
};

void check_groups(const char* what, int in, int out, int groups)
{
  if (groups <= 0 || in % groups != 0)
    throw std::runtime_error(std::string(what) + ": in_channels (" + std::to_string(in)
                             + ") must be divisible by numGroups (" + std::to_string(groups) + ")");
  if (out % groups != 0)
    throw std::runtime_error(std::string(what) + ": out_channels (" + std::to_string(out)
                             + ") must be divisible by numGroups (" + std::to_string(groups) + ")");
}

// NAM/dsp.cpp:363-398
void read_conv1x1(Conv1x1W& m, int in, int out, bool bias, int groups, WeightStream* ws)
{
  check_groups("Conv1x1", in, out, groups);
  m.in = in;
  m.out = out;
  m.groups = groups;
  m.bias = bias;
  m.w.assign((size_t)in * out, 0.0f);
  m.b.assign((size_t)out, 0.0f);
  if (!ws)
    return;
  const int opg = out / groups, ipg = in / groups;
  for (int g = 0; g < groups; g++)
    for (int i = 0; i < opg; i++)
      for (int j = 0; j < ipg; j++)
        m.w[(size_t)(g * opg + i) * in + (g * ipg + j)] = ws->next();
  if (bias)
    for (int i = 0; i < out; i++)
      m.b[i] = ws->next();
}

// NAM/conv1d.cpp:11-56 : (group, out, in, tap) with the tap index innermost
void read_conv1d(Conv1DW& m, int in, int out, int kernel, bool bias, int dilation, int groups, WeightStream* ws)
{
  check_groups("Conv1D", in, out, groups);
  if (kernel < 1 || dilation < 1)
    throw std::runtime_error("Conv1D: kernel_size and dilation must be >= 1");
  m.in = in;
  m.out = out;
  m.kernel = kernel;
  m.dilation = dilation;
  m.groups = groups;
  m.bias = bias;
  m.w.assign((size_t)kernel * in * out, 0.0f);
  m.b.assign((size_t)out, 0.0f);
  if (!ws)
    return;
  const int opg = out / groups, ipg = in / groups;
  for (int g = 0; g < groups; g++)
    for (int i = 0; i < opg; i++)
      for (int j = 0; j < ipg; j++)
        for (int k = 0; k < kernel; k++)
          m.w[((size_t)k * out + (g * opg + i)) * in + (g * ipg + j)] = ws->next();
  if (bias)
    for (int i = 0; i < out; i++)
      m.b[i] = ws->next();
}

// ---- activations (NAM/activations.cpp:55-130) -----------------------------------------------
ActType act_type_from_name(const std::string& name)
{
  static const std::pair<const char*, ActType> table[] = {
    {"Tanh", ActType::Tanh},
    {"Hardtanh", ActType::Hardtanh},
    {"Fasttanh", ActType::Fasttanh},
    {"ReLU", ActType::ReLU},
    {"LeakyReLU", ActType::LeakyReLU},
    {"PReLU", ActType::PReLU},
    {"Sigmoid", ActType::Sigmoid},
    {"SiLU", ActType::SiLU},
    {"Hardswish", ActType::Hardswish},
    {"LeakyHardtanh", ActType::LeakyHardtanh},
    {"LeakyHardTanh", ActType::LeakyHardtanh},
    {"Softsign", ActType::Softsign},
  };
  for (const auto& e : table)
    if (name == e.first)
      return e.second;
  throw std::runtime_error("Unknown activation type: " + name);
}

ActSpec parse_activation(const json::Value& j, const LoadOptions& opts)
{
  ActSpec a;
  if (j.is_null())
  {
    a.type = ActType::Identity;
    return a;
  }
  if (j.is_string())
  {
    a.type = act_type_from_name(j.as_string());
  }
  else if (j.is_object())
  {
    a.type = act_type_from_name(j.at("type").as_string("activation.type"));
    if (a.type == ActType::PReLU)
    {
      if (j.contains("negative_slope"))
        a.slopes = {(float)j.at("negative_slope").as_double()};
      else if (j.contains("negative_slopes"))
        for (const auto& v : j.at("negative_slopes").items("negative_slopes"))
          a.slopes.push_back((float)v.as_double());
    }
    else if (a.type == ActType::LeakyReLU)
      a.slope = (float)j.value_double("negative_slope", 0.01);
    else if (a.type == ActType::LeakyHardtanh)
    {
      a.min_val = (float)j.value_double("min_val", -1.0);
      a.max_val = (float)j.value_double("max_val", 1.0);
      a.min_slope = (float)j.value_double("min_slope", 0.01);
      a.max_slope = (float)j.value_double("max_slope", 0.01);
    }
  }
  else
    throw std::runtime_error("Invalid activation config: expected string or object");
  if (a.type == ActType::PReLU && a.slopes.empty())
    a.slopes = {0.01f};
  // enable_fast_tanh() swaps the "Tanh" entry of the name map (activations.cpp:168-177)
  if (opts.fast_tanh && a.type == ActType::Tanh)
    a.type = ActType::Fasttanh;
  return a;
}

Gating parse_gating(const std::string& s)
{
  if (s == "gated")
    return Gating::Gated;
  if (s == "blended")
    return Gating::Blended;
  if (s == "none")
    return Gating::None;
  throw std::runtime_error("Invalid gating_mode: " + s);
}

struct FilmParams
{
  bool active = false, shift = false;
  int groups = 1;
};

// parse_film_params, model.cpp:1190-1201
FilmParams parse_film(const json::Value& lc, const char* key)
{
  FilmParams f;
  if (!lc.contains(key))
    return f;
  const json::Value& v = lc.at(key);
  if (v.is_bool() && !v.as_bool())
    return f;
  f.active = v.value_bool("active", true);
  f.shift = v.value_bool("shift", true);
  f.groups = v.value_int("groups", 1);
  return f;
}

const char* kFilmKeys[F_COUNT] = {"conv_pre_film",       "conv_post_film",       "input_mixin_pre_film",
                                  "input_mixin_post_film", "activation_pre_film", "activation_post_film",
                                  "layer1x1_post_film",  "head1x1_post_film"};

ModelSpec build_spec(const json::Value& root, const LoadOptions& opts);

// ---- WaveNet (model.cpp:913-1276 config, :591-683 construction + weights) --------------------
void build_wavenet(ModelSpec& ms, const json::Value& config, const std::vector<float>& weights,
                   const LoadOptions& opts)
{
  WaveNetSpec& wn = ms.wavenet;
  if (config.contains("condition_dsp") && !config.at("condition_dsp").is_null())
  {
    wn.condition_dsp = std::make_shared<ModelSpec>(build_spec(config.at("condition_dsp"), opts));
    if (wn.condition_dsp->sample_rate != ms.sample_rate)
    {
      std::stringstream ss;
      ss << "Condition DSP expected sample rate (" << wn.condition_dsp->sample_rate
         << ") doesn't match WaveNet expected sample rate (" << ms.sample_rate << "!\n";
      throw std::runtime_error(ss.str());
    }
  }
  const auto& layers_json = config.at("layers").items("layers");
  if (layers_json.empty())
    throw std::runtime_error("WaveNet config requires at least one layer array");
  wn.in_channels = config.value_int("in_channels", 1);
  wn.with_head = config.contains("head") && !config.at("head").is_null();

  struct PerLayer
  {
    int kernel, dilation;
    Gating gating;
    ActSpec act, sec;
  };
  std::vector<std::vector<PerLayer>> per_layer(layers_json.size());
  std::vector<std::array<FilmParams, F_COUNT>> films(layers_json.size());

  for (size_t i = 0; i < layers_json.size(); i++)
  {
    const json::Value& lc = layers_json[i];
    const std::string where = "Layer array " + std::to_string(i);
    ArraySpec A;
    A.groups_input = lc.value_int("groups_input", 1);
    A.groups_input_mixin = lc.value_int("groups_input_mixin", 1);
    A.channels = lc.at("channels").as_int("channels");
    A.bottleneck = lc.value_int("bottleneck", A.channels);
    if (lc.contains("layer1x1"))
    {
      A.l1x1_active = lc.at("layer1x1").at("active").as_bool("layer1x1.active");
      A.l1x1_groups = lc.at("layer1x1").at("groups").as_int("layer1x1.groups");
    }
    A.input_size = lc.at("input_size").as_int("input_size");
    A.condition_size = lc.at("condition_size").as_int("condition_size");
    if (lc.contains("head") && !lc.at("head").is_null())
    {
      const json::Value& hj = lc.at("head");
      if (!hj.is_object())
        throw std::runtime_error(where + ": 'head' must be a JSON object");
      A.head_size = hj.at("out_channels").as_int("head.out_channels");
      if (hj.contains("head_dilation"))
        A.head_dilation = hj.at("head_dilation").as_int("head.head_dilation");
      A.head_kernel = hj.at("kernel_size").as_int("head.kernel_size");
      A.head_bias = hj.at("bias").as_bool("head.bias");
    }
    else if (lc.contains("head_size"))
    {
      A.head_size = lc.at("head_size").as_int("head_size");
      A.head_kernel = 1;
      A.head_bias = lc.at("head_bias").as_bool("head_bias");
    }
    else
      throw std::runtime_error(where
                               + ": expected 'head' object with out_channels, kernel_size, and bias, "
                                 "or legacy 'head_size' and 'head_bias'");
    if (A.head_kernel < 1)
      throw std::runtime_error(where + ": head.kernel_size must be >= 1");

    const auto& dil_json = lc.at("dilations").items("dilations");
    const size_t n_layers = dil_json.size();
    const bool has_k = lc.contains("kernel_size"), has_ks = lc.contains("kernel_sizes");
    std::vector<int> kernel_sizes;
    if (has_k && has_ks)
      throw std::runtime_error(where + ": only one of kernel_size (int) or kernel_sizes (array) may be provided");
    else if (has_ks)
    {
      if (!lc.at("kernel_sizes").is_array())
        throw std::runtime_error(where + ": kernel_sizes must be an array");
      for (const auto& k : lc.at("kernel_sizes").items())
        kernel_sizes.push_back(k.as_int("kernel_sizes[]"));
      if (kernel_sizes.size() != n_layers)
        throw std::runtime_error(where + ": kernel_sizes array size (" + std::to_string(kernel_sizes.size())
                                 + ") must match dilations size (" + std::to_string(n_layers) + ")");
    }
    else if (has_k)
      kernel_sizes.assign(n_layers, lc.at("kernel_size").as_int("kernel_size"));
    else
      throw std::runtime_error(where + ": either kernel_size (int) or kernel_sizes (array) must be provided");

    std::vector<ActSpec> acts;
    const json::Value& act_json = lc.at("activation");
    if (act_json.is_array())
    {
      for (const auto& a : act_json.items())
        acts.push_back(parse_activation(a, opts));
      if (acts.size() != n_layers)
        throw std::runtime_error(where + ": activation array size (" + std::to_string(acts.size())
                                 + ") must match dilations size (" + std::to_string(n_layers) + ")");
    }
    else
      acts.assign(n_layers, parse_activation(act_json, opts));

    std::vector<Gating> modes;
    std::vector<ActSpec> secs;
    const json::Value sigmoid_json = json::Value::parse("\"Sigmoid\"");
    if (lc.contains("gating_mode"))
    {
      const json::Value& gm = lc.at("gating_mode");
      const bool has_sec = lc.contains("secondary_activation");
      const json::Value& sj = lc.get("secondary_activation");
      if (gm.is_array())
      {
        for (const auto& g : gm.items())
        {
          const Gating mode = parse_gating(g.as_string("gating_mode[]"));
          modes.push_back(mode);
          if (mode != Gating::None)
          {
            if (has_sec)
            {
              if (sj.is_array())
              {
                if (modes.size() > sj.size())
                  throw std::runtime_error(where + ": secondary_activation array size must be at least "
                                           + std::to_string(modes.size()));
                secs.push_back(parse_activation(sj[modes.size() - 1], opts));
              }
              else
                secs.push_back(parse_activation(sj, opts));
            }
            else
              secs.push_back(parse_activation(sigmoid_json, opts));
          }
          else
            secs.push_back(ActSpec{});
        }
        if (modes.size() != n_layers)
          throw std::runtime_error(where + ": gating_mode array size (" + std::to_string(modes.size())
                                   + ") must match dilations size (" + std::to_string(n_layers) + ")");
        if (has_sec && sj.is_array() && sj.size() != n_layers)
          throw std::runtime_error(where + ": secondary_activation array size (" + std::to_string(sj.size())
                                   + ") must match dilations size (" + std::to_string(n_layers) + ")");
      }
      else
      {
        const Gating mode = parse_gating(gm.as_string("gating_mode"));
        modes.assign(n_layers, mode);
        ActSpec sec;
        if (mode != Gating::None)
          sec = has_sec ? parse_activation(sj, opts) : parse_activation(sigmoid_json, opts);
        secs.assign(n_layers, sec);
      }
    }
    else if (lc.contains("gated"))
    {
      const bool gated = lc.at("gated").as_bool("gated");
      modes.assign(n_layers, gated ? Gating::Gated : Gating::None);
      secs.assign(n_layers, gated ? parse_activation(sigmoid_json, opts) : ActSpec{});
    }
    else
    {
      modes.assign(n_layers, Gating::None);
      secs.assign(n_layers, ActSpec{});
    }

    A.h1x1_out = A.channels;
    if (lc.contains("head1x1"))
    {
      const json::Value& h = lc.at("head1x1");
      A.h1x1_active = h.at("active").as_bool("head1x1.active");
      A.h1x1_out = h.at("out_channels").as_int("head1x1.out_channels");
      A.h1x1_groups = h.at("groups").as_int("head1x1.groups");
    }
    for (int f = 0; f < F_COUNT; f++)
      films[i][f] = parse_film(lc, kFilmKeys[f]);
    if (films[i][F_L1X1_POST].active && !A.l1x1_active)
      throw std::runtime_error(where + ": layer1x1_post_film cannot be active when layer1x1.active is false");

    for (size_t l = 0; l < n_layers; l++)
      per_layer[i].push_back(PerLayer{kernel_sizes[l], dil_json[l].as_int("dilations[]"), modes[l], acts[l], secs[l]});
    wn.arrays.push_back(std::move(A));
  }

  // Constructor-time validation (model.cpp:596-651, detail.h:56-90)
  if (wn.condition_dsp)
  {
    if (wn.in_channels != wn.condition_dsp->in_channels)
      throw std::runtime_error("input channels of WaveNet (" + std::to_string(wn.in_channels)
                               + ") don't match input channels of condition DSP ("
                               + std::to_string(wn.condition_dsp->in_channels) + "!\n");
    for (size_t i = 0; i < wn.arrays.size(); i++)
      if (wn.arrays[i].condition_size != wn.condition_dsp->out_channels)
        throw std::runtime_error("condition_size of layer " + std::to_string(i) + " ("
                                 + std::to_string(wn.arrays[i].condition_size)
                                 + ") doesn't match output channels of condition DSP ("
                                 + std::to_string(wn.condition_dsp->out_channels) + "!\n");
  }
  for (size_t i = 1; i < wn.arrays.size(); i++)
  {
    if (wn.arrays[i].channels != wn.arrays[i - 1].head_size)
      throw std::runtime_error("channels of layer " + std::to_string(i) + " (" + std::to_string(wn.arrays[i].channels)
                               + ") doesn't match head_size of preceding layer ("
                               + std::to_string(wn.arrays[i - 1].head_size) + "!\n");
    // The head accumulator of array i is initialised by a straight copy of array i-1's head
    // output (model.cpp:473-486), so the row counts must agree.
    if (wn.arrays[i].head_out_size() != wn.arrays[i - 1].head_size)
      throw std::runtime_error("layer array " + std::to_string(i) + ": head accumulator rows ("
                               + std::to_string(wn.arrays[i].head_out_size()) + ") != previous head_size ("
                               + std::to_string(wn.arrays[i - 1].head_size) + ")");
  }

  PostHeadSpec& ph = wn.post_head;
  std::vector<int> ph_kernels;
  if (wn.with_head)
  {
    const json::Value& hj = config.at("head");
    const int implied_in = wn.arrays.back().head_size;
    if (hj.contains("in_channels") && !hj.at("in_channels").is_null()
        && hj.at("in_channels").as_int("head.in_channels") != implied_in)
      throw std::runtime_error("WaveNet config: head.in_channels (" + std::to_string(hj.at("in_channels").as_int())
                               + ") must equal last layer's head_size (" + std::to_string(implied_in) + ")");
    ph.in_channels = implied_in;
    ph.channels = hj.at("channels").as_int("head.channels");
    ph.out_channels = hj.at("out_channels").as_int("head.out_channels");
    for (const auto& k : hj.at("kernel_sizes").items("head.kernel_sizes"))
      ph_kernels.push_back(k.as_int());
    ph.act = parse_activation(hj.at("activation"), opts);
    if (ph_kernels.empty())
      throw std::runtime_error("WaveNet config: head.kernel_sizes must be non-empty");
    for (int k : ph_kernels)
      if (k < 1)
        throw std::runtime_error("WaveNet Head: kernel_sizes entries must be >= 1");
  }

  // ---- weights, in stream order (model.cpp:661-670, :563-569, :152-181) ----
  WeightStream ws(weights);
  for (size_t i = 0; i < wn.arrays.size(); i++)
  {
    ArraySpec& A = wn.arrays[i];
    read_conv1x1(A.rechannel, A.input_size, A.channels, false, 1, &ws);
    for (const PerLayer& pl : per_layer[i])
    {
      LayerSpec L;
      L.gating = pl.gating;
      L.act = pl.act;
      L.sec_act = pl.sec;
      const int zrows = (pl.gating != Gating::None) ? 2 * A.bottleneck : A.bottleneck;
      L.has_l1x1 = A.l1x1_active;
      L.has_h1x1 = A.h1x1_active;
      if (!A.l1x1_active && A.bottleneck != A.channels)
        throw std::invalid_argument("When layer1x1.active is false, bottleneck (" + std::to_string(A.bottleneck)
                                    + ") must equal channels (" + std::to_string(A.channels) + ")");
      if (!A.h1x1_active && films[i][F_H1X1_POST].active)
        throw std::invalid_argument("Do not use post-head 1x1 FiLM if there is no head 1x1");
      read_conv1d(L.conv, A.channels, zrows, pl.kernel, true, pl.dilation, A.groups_input, &ws);
      read_conv1x1(L.mixin, A.condition_size, zrows, false, A.groups_input_mixin, &ws);
      if (L.has_l1x1)
        read_conv1x1(L.l1x1, A.bottleneck, A.channels, true, A.l1x1_groups, &ws);
      if (L.has_h1x1)
        read_conv1x1(L.h1x1, A.bottleneck, A.h1x1_out, true, A.h1x1_groups, &ws);
      const int dims[F_COUNT] = {A.channels, zrows, A.condition_size, zrows, zrows, A.bottleneck, A.channels,
                                 A.h1x1_out};
      for (int f = 0; f < F_COUNT; f++)
      {
        FilmSpec& fs = L.film[f];
        fs.active = films[i][f].active;
        if (f == F_L1X1_POST && !A.l1x1_active)
          fs.active = false;
        if (f == F_H1X1_POST && !A.h1x1_active)
          fs.active = false;
        if (!fs.active)
          continue;
        fs.shift = films[i][f].shift;
        fs.groups = films[i][f].groups;
        fs.dim = dims[f];
        read_conv1x1(fs.css, A.condition_size, (fs.shift ? 2 : 1) * fs.dim, true, fs.groups, &ws);
      }
      A.layers.push_back(std::move(L));
    }
    // LayerArray ctor (model.cpp:397-400): Conv1D(head_out_size -> head_size, head_kernel, head_bias, head_dilation)
    read_conv1d(A.head_rechannel, A.head_out_size(), A.head_size, A.head_kernel, A.head_bias, A.head_dilation, 1, &ws);
  }
  if (wn.with_head)
  {
    int cin = ph.in_channels;
    for (size_t i = 0; i < ph_kernels.size(); i++)
    {
      const int cout = (i + 1 == ph_kernels.size()) ? ph.out_channels : ph.channels;
      Conv1DW c;
      read_conv1d(c, cin, cout, ph_kernels[i], true, 1, 1, &ws);
      ph.convs.push_back(std::move(c));
      cin = cout;
    }
  }
  wn.head_scale = ws.next();
  if (ws.position() != ws.size())
    throw std::runtime_error("Weight mismatch: assigned " + std::to_string(ws.position()) + " weights, but "
                             + std::to_string(ws.size()) + " were provided.");

  ms.in_channels = wn.in_channels;
  ms.out_channels = wn.with_head ? ph.out_channels : wn.arrays.back().head_size;
  // model.cpp:653-658
  long pw = wn.condition_dsp ? wn.condition_dsp->prewarm_samples : 1;
  for (const auto& A : wn.arrays)
    pw += A.receptive_field();
  if (wn.with_head)
  {
    long rf = 1;
    for (const auto& c : ph.convs)
      rf += c.kernel - 1;
    pw += rf - 1;
  }
  ms.prewarm_samples = (int)pw;
}

void build_lstm(ModelSpec& ms, const json::Value& config, const std::vector<float>& weights)
{
  LstmSpec& ls = ms.lstm;
  ls.num_layers = config.at("num_layers").as_int("num_layers");
  ls.input_size = config.at("input_size").as_int("input_size");
  ls.hidden = config.at("hidden_size").as_int("hidden_size");
  ms.in_channels = config.value_int("in_channels", 1);
  ms.out_channels = config.value_int("out_channels", 1);
  if (ls.num_layers < 0 || ls.hidden <= 0 || ls.input_size <= 0)
    throw std::runtime_error("LSTM: bad configuration");
  WeightStream ws(weights);
  const int H = ls.hidden;
  for (int l = 0; l < ls.num_layers; l++)
  {
    LstmCellW c;
    c.input_size = (l == 0) ? ls.input_size : H;
    c.hidden = H;
    const int W = c.input_size + H;
    c.w.resize((size_t)4 * H * W);
    for (auto& v : c.w)
      v = ws.next();
    c.b.resize((size_t)4 * H);
    for (auto& v : c.b)
      v = ws.next();
    c.h0.resize(H);
    for (auto& v : c.h0)
      v = ws.next();
    c.c0.resize(H);
    for (auto& v : c.c0)
      v = ws.next();
    ls.cells.push_back(std::move(c));
  }
  ls.head_w.resize((size_t)ms.out_channels * H);
  for (auto& v : ls.head_w)
    v = ws.next();
  ls.head_b.resize((size_t)ms.out_channels);
  for (auto& v : ls.head_b)
    v = ws.next();
  if (ws.position() != ws.size())
    throw std::runtime_error("LSTM weight mismatch: assigned " + std::to_string(ws.position()) + " weights, but "
                             + std::to_string(ws.size()) + " were provided.");
  // lstm.cpp:127-134
  const int pw = (int)(0.5 * ms.sample_rate);
  ms.prewarm_samples = pw <= 0 ? 1 : pw;
}

void build_linear(ModelSpec& ms, const json::Value& config, const std::vector<float>& weights)
{
  LinearSpec& li = ms.linear;
  li.receptive_field = config.at("receptive_field").as_int("receptive_field");
  li.bias = config.at("bias").as_bool("bias");
  // "implementation" (linear.cpp:280-293): auto / direct / fft pick HOW the reference evaluates the same FIR (direct form
  // or partitioned FFT above 256 taps); the result is the same, and the CUDA path always runs direct form.  Unknown
  // names are rejected like the reference does.
  if (config.contains("implementation"))
  {
    std::string impl = config.at("implementation").as_string("implementation");
    for (char& ch : impl)
      ch = (char)std::tolower((unsigned char)ch);
    static const char* known[] = {"auto", "direct", "legacy", "old", "fft", "partitioned_fft", "partitioned-fft"};
    bool ok = false;
    for (const char* k : known)
      ok = ok || impl == k;
    if (!ok)
      throw std::runtime_error("Unsupported Linear implementation: " + config.at("implementation").as_string("implementation"));
  }
  ms.in_channels = config.value_int("in_channels", 1);
  ms.out_channels = config.value_int("out_channels", 1);
  if (li.receptive_field <= 0)
    throw std::runtime_error("Linear: receptive_field must be positive");
  if ((int)weights.size() != li.receptive_field + (li.bias ? 1 : 0))
    throw std::runtime_error("Params vector does not match expected size based on architecture parameters");
  li.impulse.assign(weights.begin(), weights.begin() + li.receptive_field);
  li.bias_value = li.bias ? weights[li.receptive_field] : 0.0f;
  ms.prewarm_samples = 0;
}

// NAM/convnet.cpp:321-335 (config), :172-201 (constructor), :48-60 (block), :14-37 (BatchNorm), :132-153 (head)
void build_convnet(ModelSpec& ms, const json::Value& config, const std::vector<float>& weights, const LoadOptions& opts)
{
  ConvNetSpec& cn = ms.convnet;
  cn.channels = config.at("channels").as_int("channels");
  cn.batchnorm = config.at("batchnorm").as_bool("batchnorm");
  cn.groups = config.value_int("groups", 1);
  cn.act = parse_activation(config.at("activation"), opts);
  ms.in_channels = config.value_int("in_channels", 1);
  ms.out_channels = config.value_int("out_channels", 1);
  if (cn.channels <= 0 || ms.in_channels <= 0 || ms.out_channels <= 0)
    throw std::runtime_error("ConvNet: bad configuration");
  std::vector<int> dilations;
  for (const auto& d : config.at("dilations").items("dilations"))
    dilations.push_back(d.as_int("dilations[]"));
  if (dilations.empty())
    throw std::runtime_error("ConvNet: 'dilations' must not be empty");
  WeightStream ws(weights);
  const int C = cn.channels;
  long pw = 1; // convnet.cpp:198-200
  for (size_t i = 0; i < dilations.size(); i++)
  {
    ConvNetSpec::Block b;
    read_conv1d(b.conv, i == 0 ? ms.in_channels : C, C, 2, !cn.batchnorm, dilations[i], cn.groups, &ws);
    if (cn.batchnorm)
    {
      std::vector<float> mean(C), var(C), w(C), bias(C);
      for (auto& v : mean)
        v = ws.next();
      for (auto& v : var)
        v = ws.next();
      for (auto& v : w)
        v = ws.next();
      for (auto& v : bias)
        v = ws.next();
      const float eps = ws.next();
      b.scale.resize(C);
      b.loc.resize(C);
      for (int j = 0; j < C; j++)
      {
        b.scale[j] = w[j] / std::sqrt(eps + var[j]);
        b.loc[j] = bias[j] - b.scale[j] * mean[j];
      }
    }
    pw += dilations[i];
    cn.blocks.push_back(std::move(b));
  }
  read_conv1x1(cn.head, C, ms.out_channels, true, 1, &ws);
  if (ws.position() != ws.size())
    throw std::runtime_error("Didn't touch all the weights when initializing ConvNet");
  ms.prewarm_samples = (int)pw;
}


// ---- "slimmable" WaveNet (model.cpp:1290-1315 dispatch; NAM/wavenet/slimmable.cpp) ----------------------------
// A WaveNet whose layer arrays carry {"slimmable": {"method": "slice_channels_uniform", ...}} is, in the reference,
// a SlimmableWavenet: SetSlimmableSize(ratio) picks a channel count per array from its allowed_channels, keeps the
// FIRST rows / columns of every weight tensor and builds a fresh, smaller WaveNet.  Here it becomes a container of
// plain WaveNet documents, one per interval between the ratio breakpoints, so the SlimmableContainer machinery
// (create_common, nam_b200_set_slimmable_size) serves it unchanged.
bool config_is_slimmable_wavenet(const json::Value& config)
{
  if (!config.is_object() || !config.contains("layers") || !config.at("layers").is_array())
    return false;
  for (const auto& lc : config.at("layers").items("layers"))
  {
    if (!lc.is_object() || !lc.contains("slimmable") || !lc.at("slimmable").is_object())
      continue;
    const json::Value& m = lc.at("slimmable").get("method");
    const std::string method = m.is_string() ? m.as_string() : std::string();
    if (method != "slice_channels_uniform")
    {
      if (!method.empty())
        throw std::runtime_error("SlimmableWavenet: unsupported slimmable method '" + method + "'");
      continue;
    }
    return true;
  }
  return false;
}

// reads the full weight stream tensor by tensor and keeps the leading rows / columns (slimmable.cpp:20-69)
class WeightSlicer
{
public:
  WeightSlicer(const std::vector<float>& full, std::vector<float>& slim)
  : _full(full)
  , _slim(slim)
  {
  }
  // (out x in x taps) weights, tap innermost, then an optional bias of `out`
  void tensor(int out, int in, int taps, int keep_out, int keep_in, bool bias)
  {
    for (int o = 0; o < out; o++)
      for (int i = 0; i < in; i++)
        for (int k = 0; k < taps; k++)
        {
          const float w = next();
          if (o < keep_out && i < keep_in)
            _slim.push_back(w);
        }
    if (bias)
      for (int o = 0; o < out; o++)
      {
        const float b = next();
        if (o < keep_out)
          _slim.push_back(b);
      }
  }
  void copy(int n)
  {
    for (int i = 0; i < n; i++)
      _slim.push_back(next());
  }
  bool done() const { return _pos == _full.size(); }

private:
  float next()
  {
    if (_pos >= _full.size())
      throw std::runtime_error("SlimmableWavenet: weight stream too short");
    return _full[_pos++];
  }
  const std::vector<float>& _full;
  std::vector<float>& _slim;
  size_t _pos = 0;
};

int slim_bottleneck(const ArraySpec& A, int new_channels)
{
  if (!A.l1x1_active)
    return new_channels; // bottleneck must equal channels when layer1x1 is inactive (slimmable.cpp:81-86)
  return std::max(1, A.bottleneck * new_channels / A.channels);
}

// extract_slimmed_weights (slimmable.cpp:133-262), in the weight-stream order of the WaveNet constructor
std::vector<float> slice_wavenet_weights(const WaveNetSpec& wn, const std::vector<float>& full, const std::vector<int>& target)
{
  std::vector<float> slim;
  WeightSlicer ws(full, slim);
  const int n_arrays = (int)wn.arrays.size();
  for (int a = 0; a < n_arrays; a++)
  {
    const ArraySpec& A = wn.arrays[(size_t)a];
    if (A.head_kernel != 1)
      throw std::runtime_error("SlimmableWavenet: head rechannel kernel_size must be 1 (slimming with head kernel_size > 1 "
                               "is not implemented)");
    if (A.groups_input != 1)
      throw std::runtime_error("SlimmableWavenet: groups_input > 1 not supported");
    if (A.groups_input_mixin != 1)
      throw std::runtime_error("SlimmableWavenet: groups_input_mixin > 1 not supported");
    if (A.l1x1_active && A.l1x1_groups != 1)
      throw std::runtime_error("SlimmableWavenet: layer1x1 groups > 1 not supported");
    if (A.h1x1_active && A.h1x1_groups != 1)
      throw std::runtime_error("SlimmableWavenet: head1x1 groups > 1 not supported");
    const int C = A.channels, B = A.bottleneck, c = target[(size_t)a], b = slim_bottleneck(A, c), cond = A.condition_size;
    const int in_keep = (a == 0) ? A.input_size : target[(size_t)a - 1];
    const int head_keep = (a + 1 < n_arrays) ? target[(size_t)a + 1] : A.head_size;
    const int HO = A.h1x1_active ? A.h1x1_out : B, ho = A.h1x1_active ? A.h1x1_out : b;
    ws.tensor(C, A.input_size, 1, c, in_keep, false); // rechannel
    for (const LayerSpec& L : A.layers)
    {
      const int mult = (L.gating != Gating::None) ? 2 : 1;
      const int BG = mult * B, bg = mult * b;
      ws.tensor(BG, C, L.conv.kernel, bg, c, true); // conv
      ws.tensor(BG, cond, 1, bg, cond, false); // input mixin
      if (A.l1x1_active)
        ws.tensor(C, B, 1, c, b, true);
      if (A.h1x1_active)
        ws.tensor(A.h1x1_out, B, 1, A.h1x1_out, b, true);
      // the eight FiLM sites in weight-stream order; the kept rows are the LEADING rows of the (scale | shift) stack,
      // exactly as the reference slices them (slimmable.cpp:186-254)
      const int full_dim[F_COUNT] = {C, BG, cond, BG, BG, B, C, A.h1x1_out};
      const int keep_dim[F_COUNT] = {c, bg, cond, bg, bg, b, c, A.h1x1_out};
      for (int f = 0; f < F_COUNT; f++)
      {
        const FilmSpec& F = L.film[f];
        if (!F.active || (f == F_L1X1_POST && !A.l1x1_active) || (f == F_H1X1_POST && !A.h1x1_active))
          continue;
        const int m2 = F.shift ? 2 : 1;
        ws.tensor(m2 * full_dim[f], cond, 1, m2 * keep_dim[f], cond, true);
      }
    }
    ws.tensor(A.head_size, HO, 1, head_keep, ho, A.head_bias); // head rechannel
  }
  ws.copy(1); // head_scale
  if (!ws.done())
    throw std::runtime_error("SlimmableWavenet: weight stream longer than the configuration implies");
  return slim;
}

std::string json_number(double v)
{
  return json::number_to_string(v); // locale-independent
}

// one layer-array config with its channel counts replaced and "slimmable" cleared (modify_params_for_channels,
// slimmable.cpp:268-295)
std::string slim_layer_json(const json::Value& lc, int channels, int bottleneck, int input_size, int head_size)
{
  std::string out = "{";
  bool first = true, saw_bottleneck = false;
  auto emit = [&](const std::string& key, const std::string& value) {
    out += (first ? "\"" : ", \"") + key + "\": " + value;
    first = false;
  };
  for (const auto& kv : lc.members())
  {
    if (kv.first == "channels")
      emit(kv.first, std::to_string(channels));
    else if (kv.first == "bottleneck")
    {
      emit(kv.first, std::to_string(bottleneck));
      saw_bottleneck = true;
    }
    else if (kv.first == "input_size")
      emit(kv.first, std::to_string(input_size));
    else if (kv.first == "head_size")
      emit(kv.first, std::to_string(head_size));
    else if (kv.first == "slimmable")
      emit(kv.first, "null");
    else if (kv.first == "head" && kv.second.is_object())
    {
      std::string h = "{";
      bool hf = true;
      for (const auto& hk : kv.second.members())
      {
        h += (hf ? "\"" : ", \"") + hk.first + "\": " + (hk.first == "out_channels" ? std::to_string(head_size) : hk.second.dump());
        hf = false;
      }
      emit(kv.first, h + "}");
    }
    else
      emit(kv.first, kv.second.dump());
  }
  if (!saw_bottleneck)
    emit("bottleneck", std::to_string(bottleneck));
  return out + "}";
}

void build_slimmable_wavenet(ModelSpec& ms, const json::Value& root, const json::Value& config,
                             const std::vector<float>& weights, const LoadOptions& opts)
{
  // the full-size network: validates the configuration and the weight count, gives every tensor's dimensions
  ModelSpec full = ms;
  build_wavenet(full, config, weights, opts);
  const WaveNetSpec& wn = full.wavenet;
  const auto& layers_json = config.at("layers").items("layers");
  const size_t n_arrays = wn.arrays.size();
  // per-array allowed channel counts (SlimmableWavenetConfig::create, slimmable.cpp:540-571)
  std::vector<std::vector<int>> allowed(n_arrays);
  bool any = false;
  for (size_t i = 0; i < n_arrays; i++)
  {
    const json::Value& lc = layers_json[i];
    if (!lc.contains("slimmable") || !lc.at("slimmable").is_object())
      continue;
    const json::Value& sc = lc.at("slimmable");
    const json::Value& mj = sc.get("method");
    const std::string method = mj.is_string() ? mj.as_string() : std::string();
    if (method != "slice_channels_uniform")
      throw std::runtime_error("SlimmableWavenet: unsupported slimmable method '" + method + "'");
    const json::Value& kw = sc.get("kwargs");
    if (kw.is_object() && kw.contains("allowed_channels"))
      for (const auto& ch : kw.at("allowed_channels").items("allowed_channels"))
        allowed[i].push_back(ch.as_int("allowed_channels[]"));
    else
      for (int c = 1; c <= wn.arrays[i].channels; c++)
        allowed[i].push_back(c);
    // constructor checks (slimmable.cpp:368-388)
    for (size_t j = 1; j < allowed[i].size(); j++)
      if (allowed[i][j] <= allowed[i][j - 1])
        throw std::runtime_error("SlimmableWavenet: allowed_channels must be sorted ascending");
    if (!allowed[i].empty())
    {
      any = true;
      if (allowed[i].back() != wn.arrays[i].channels)
        throw std::runtime_error(
          "SlimmableWavenet: last allowed_channels entry must equal the full channel count for that array");
      if (allowed[i].front() < 1)
        throw std::runtime_error("SlimmableWavenet: allowed_channels must be positive");
    }
  }
  if (!any)
    throw std::runtime_error("SlimmableWavenet: at least one layer array must have allowed_channels");
  if (wn.with_head)
    throw std::runtime_error("SlimmableWavenet: post-stack head is not supported");

  // ratio breakpoints i / len over all arrays (get_ratio_breakpoints, slimmable.cpp:111-125)
  std::vector<double> bps;
  for (const auto& al : allowed)
    for (size_t i = 1; i < al.size(); i++)
      bps.push_back((double)i / (double)al.size());
  std::sort(bps.begin(), bps.end());
  bps.erase(std::unique(bps.begin(), bps.end()), bps.end());
  auto channels_at = [&](double ratio) { // ratio_to_channels (slimmable.cpp:104-109) per array
    std::vector<int> t(n_arrays);
    for (size_t i = 0; i < n_arrays; i++)
    {
      const auto& al = allowed[i];
      if (al.empty())
        t[i] = wn.arrays[i].channels;
      else
        t[i] = al[(size_t)std::min((int)std::floor(ratio * (double)al.size()), (int)al.size() - 1)];
    }
    return t;
  };

  ms.arch = Arch::Container;
  ms.in_channels = full.in_channels;
  ms.out_channels = full.out_channels;
  ms.prewarm_samples = 0; // SlimmableWavenet::GetPrewarmSamples (slimmable.h:71): the active model prewarms itself
  for (size_t k = 0; k <= bps.size(); k++)
  {
    const double lo = (k == 0) ? 0.0 : bps[k - 1], hi = (k == bps.size()) ? 1.0 : bps[k];
    const std::vector<int> target = channels_at(0.5 * (lo + hi));
    ModelSpec::Submodel sm;
    // nam_b200_set_slimmable_size picks the first sub-model with value < max_value; the reference evaluates
    // floor(value * len) at the breakpoint itself: where rounding puts that below the breakpoint's own index the
    // breakpoint value still belongs to this interval
    sm.max_value = (k == bps.size()) ? 1.0 : hi;
    if (k < bps.size() && channels_at(hi) == target)
      sm.max_value = std::nextafter(hi, 2.0);
    bool is_full = true;
    for (size_t i = 0; i < n_arrays; i++)
      is_full = is_full && target[i] == wn.arrays[i].channels;
    const std::vector<float> w = is_full ? weights : slice_wavenet_weights(wn, weights, target);
    std::string cfg = "{";
    bool first = true;
    for (const auto& kv : config.members())
    {
      cfg += first ? "\"" : ", \"";
      first = false;
      cfg += kv.first + "\": ";
      if (kv.first != "layers")
      {
        cfg += kv.second.dump();
        continue;
      }
      cfg += "[";
      for (size_t i = 0; i < n_arrays; i++)
      {
        const ArraySpec& A = wn.arrays[i];
        const int in_size = (i == 0) ? A.input_size : target[i - 1];
        const int head_size = (i + 1 < n_arrays) ? target[i + 1] : A.head_size;
        cfg += (i ? ", " : "") + slim_layer_json(layers_json[i], target[i], slim_bottleneck(A, target[i]), in_size, head_size);
      }
      cfg += "]";
    }
    cfg += "}";
    std::string doc = "{";
    for (const auto& kv : root.members())
      if (kv.first != "config" && kv.first != "weights")
        doc += "\"" + kv.first + "\": " + kv.second.dump() + ", ";
    doc += "\"config\": " + cfg + ", \"weights\": [";
    for (size_t i = 0; i < w.size(); i++)
    {
      doc += (i ? ", " : "") + json::number_to_string((double)w[i]); // exact and locale-independent
    }
    doc += "]}";
    sm.model_json = std::move(doc);
    ms.submodels.push_back(std::move(sm));
  }
}

// ---- model fingerprint (ModelSpec::fingerprint) ----------------------------------------------
struct Fnv64
{
  uint64_t h = 0xcbf29ce484222325ull;
  void bytes(const void* p, size_t n)
  {
    const unsigned char* c = static_cast<const unsigned char*>(p);
    for (size_t i = 0; i < n; i++)
      h = (h ^ c[i]) * 0x100000001b3ull;
  }
  void u64(uint64_t v) { bytes(&v, sizeof v); }
  void str(const std::string& s)
  {
    u64(s.size());
    bytes(s.data(), s.size());
  }
  // canonical walk: a type tag per value, object members in key order
  void value(const json::Value& v)
  {
    u64((uint64_t)v.type());
    switch (v.type())
    {
      case json::Value::Type::Null: break;
      case json::Value::Type::Bool: u64(v.as_bool() ? 1 : 0); break;
      case json::Value::Type::Number:
      {
        const double d = v.as_double();
        bytes(&d, sizeof d);
        break;
      }
      case json::Value::Type::String: str(v.as_string()); break;
      case json::Value::Type::Array:
        u64(v.size());
        for (const auto& item : v.items())
          value(item);
        break;
      case json::Value::Type::Object:
      {
        std::vector<const std::pair<std::string, json::Value>*> members;
        for (const auto& kv : v.members())
          members.push_back(&kv);
        std::sort(members.begin(), members.end(), [](auto* a, auto* b) { return a->first < b->first; });
        u64(members.size());
        for (auto* kv : members)
        {
          str(kv->first);
          value(kv->second);
        }
        break;
      }
    }
  }
};

uint64_t model_fingerprint(const std::string& architecture, const json::Value& config, const std::vector<float>& weights)
{
  Fnv64 f;
  f.str(architecture);
  f.value(config);
  f.u64(weights.size());
  f.bytes(weights.data(), weights.size() * sizeof(float));
  return f.h;
}

// the same over the architecture and the "config" object alone, without its "head_scale" field (the reference reads the
// scale from the last weight, model.cpp:670): equal for documents that differ in their weights only.  A nested
// "condition_dsp" document contributes its architecture, its sample rate and its own config fingerprint: its weights,
// metadata and version are the sub-model's data, like the outer document's.
uint64_t config_fingerprint(const std::string& architecture, const json::Value& config)
{
  Fnv64 f;
  f.str(architecture);
  if (!config.is_object())
  {
    f.value(config);
    return f.h;
  }
  std::vector<const std::pair<std::string, json::Value>*> members;
  for (const auto& kv : config.members())
    if (kv.first != "head_scale")
      members.push_back(&kv);
  std::sort(members.begin(), members.end(), [](auto* a, auto* b) { return a->first < b->first; });
  f.u64(members.size());
  for (auto* kv : members)
  {
    f.str(kv->first);
    const json::Value& v = kv->second;
    if (kv->first == "condition_dsp" && v.is_object() && v.contains("architecture") && v.contains("config"))
    {
      const json::Value& arch = v.at("architecture");
      f.value(arch);
      f.value(v.get("sample_rate"));
      f.u64(config_fingerprint(arch.is_string() ? arch.as_string() : std::string(), v.at("config")));
    }
    else
      f.value(v);
  }
  return f.h;
}

ModelSpec build_spec(const json::Value& root, const LoadOptions& opts)
{
  if (!root.is_object())
    throw std::runtime_error("Invalid .nam: root JSON value must be an object.");
  static const char* required[] = {"version", "architecture", "config", "weights"};
  for (const char* key : required)
    if (!root.contains(key))
      throw std::runtime_error(std::string("Invalid .nam: missing required key \"") + key + "\".");
  ModelSpec ms;
  ms.version = root.at("version").as_string("version");
  const VersionSupport sup = version_support(ms.version);
  if (sup == VersionSupport::No)
    throw std::runtime_error("Model config is an unsupported version " + ms.version + ".");
  if (sup == VersionSupport::Partial)
    std::cerr << "Model config is a partially-supported version " << ms.version << ". Continuing with partial support."
              << std::endl;
  ms.architecture = root.at("architecture").as_string("architecture");
  ms.sample_rate = root.contains("sample_rate") ? root.at("sample_rate").as_double("sample_rate") : -1.0;
  std::vector<float> weights;
  {
    const auto& wj = root.at("weights").items("weights");
    weights.reserve(wj.size());
    for (const auto& v : wj)
      weights.push_back((float)v.as_double("weights[]"));
  }
  ms.n_weights = weights.size();
  const json::Value& md = root.get("metadata");
  if (md.is_object())
  {
    auto extract = [&md](const char* key) -> std::optional<double> {
      if (md.contains(key) && !md.at(key).is_null())
        return md.at(key).as_double(key);
      return std::nullopt;
    };
    ms.loudness = extract("loudness");
    ms.input_level = extract("input_level_dbu");
    ms.output_level = extract("output_level_dbu");
  }
  const json::Value& config = root.at("config");
  ms.fingerprint = model_fingerprint(ms.architecture, config, weights);
  ms.config_fingerprint = config_fingerprint(ms.architecture, config);
  if (ms.architecture == "WaveNet" && config_is_slimmable_wavenet(config))
    build_slimmable_wavenet(ms, root, config, weights, opts);
  else if (ms.architecture == "WaveNet")
  {
    ms.arch = Arch::WaveNet;
    build_wavenet(ms, config, weights, opts);
  }
  else if (ms.architecture == "LSTM")
  {
    ms.arch = Arch::LSTM;
    build_lstm(ms, config, weights);
  }
  else if (ms.architecture == "Linear")
  {
    ms.arch = Arch::Linear;
    build_linear(ms, config, weights);
  }
  else if (ms.architecture == "ConvNet")
  {
    ms.arch = Arch::ConvNet;
    build_convnet(ms, config, weights, opts);
  }
  else if (ms.architecture == "SlimmableContainer")
  {
    // ContainerConfig::create + ContainerModel ctor (container.cpp:19-47,146-169): the container has no
    // weights of its own, every entry of config.submodels is {max_value, model: <a whole .nam document>}
    ms.arch = Arch::Container;
    const json::Value& subs = config.get("submodels");
    if (!subs.is_array() || subs.size() == 0)
      throw std::runtime_error("SlimmableContainer: 'submodels' must be a non-empty array");
    for (const auto& entry : subs.items("submodels"))
    {
      ModelSpec::Submodel sm;
      sm.max_value = entry.at("max_value").as_double("max_value");
      sm.model_json = entry.at("model").dump();
      ms.submodels.push_back(std::move(sm));
    }
    for (size_t i = 1; i < ms.submodels.size(); i++)
      if (ms.submodels[i].max_value <= ms.submodels[i - 1].max_value)
        throw std::runtime_error("ContainerModel: submodels must be sorted by ascending max_value");
    if (ms.submodels.back().max_value < 1.0)
      throw std::runtime_error("ContainerModel: last submodel max_value must be >= 1.0");
  }
  else
    throw std::runtime_error("No config parser registered for architecture: " + ms.architecture);
  if (ms.in_channels <= 0 || ms.out_channels <= 0)
    throw std::runtime_error("Channel counts must be positive");
  return ms;
}

} // namespace

long ArraySpec::receptive_field() const
{
  long r = 0;
  for (const auto& L : layers)
    r += L.conv.lookback();
  r += head_rechannel.lookback();
  return r;
}

// NAM/get_dsp.cpp:18-39; versions: 0.5.0 <= v, same major/minor <= 0.7, later patch = partial
VersionSupport version_support(const std::string& version)
{
  int parts[3] = {0, 0, 0};
  size_t pos = 0;
  for (int p = 0; p < 3; p++)
  {
    if (pos >= version.size() || !std::isdigit((unsigned char)version[pos]))
      return VersionSupport::No;
    long v = 0;
    while (pos < version.size() && std::isdigit((unsigned char)version[pos]))
    {
      v = v * 10 + (version[pos] - '0');
      if (v > 1000000)
        return VersionSupport::No;
      pos++;
    }
    parts[p] = (int)v;
    if (p < 2)
    {
      if (pos >= version.size() || version[pos] != '.')
        return VersionSupport::No;
      pos++;
    }
  }
  if (pos != version.size())
    return VersionSupport::No;
  const int latest[3] = {0, 7, 0}, earliest[3] = {0, 5, 0};
  auto less = [](const int* a, const int* b) {
    return a[0] < b[0] || (a[0] == b[0] && (a[1] < b[1] || (a[1] == b[1] && a[2] < b[2])));
  };
  if (less(parts, earliest))
    return VersionSupport::No;
  if (parts[0] > latest[0] || parts[1] > latest[1])
    return VersionSupport::No;
  if (less(latest, parts))
    return VersionSupport::Partial;
  return VersionSupport::Yes;
}

ModelSpec model_spec_from_json(const json::Value& root, const LoadOptions& opts)
{
  return build_spec(root, opts);
}

ModelSpec model_spec_from_text(const std::string& text, const LoadOptions& opts)
{
  return build_spec(json::Value::parse(text), opts);
}

ModelSpec model_spec_from_file(const std::string& path, const LoadOptions& opts)
{
  std::ifstream in(path, std::ios::binary);
  if (!in.is_open())
  {
    std::ifstream probe(path);
    throw NamFileValidationError("Could not validate .nam file [" + path + "]: "
                                 + (probe.good() ? "file could not be read." : "file does not exist."));
  }
  std::stringstream ss;
  ss << in.rdbuf();
  json::Value root;
  try
  {
    root = json::Value::parse(ss.str());
  }
  catch (const json::ParseError& e)
  {
    throw NamFileValidationError("Could not parse .nam file [" + path + "]: " + e.what());
  }
  if (!root.is_object())
    throw NamFileValidationError("Invalid .nam file [" + path + "]: root JSON value must be an object.");
  static const char* required[] = {"version", "architecture", "config", "weights"};
  for (const char* key : required)
    if (!root.contains(key))
      throw NamFileValidationError("Invalid .nam file [" + path + "]: missing required key \"" + key + "\".");
  return build_spec(root, opts);
}

} // namespace namb200
