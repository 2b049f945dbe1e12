#include "stream_state.h"

#include <cinttypes>
#include <cstdio>
#include <cstring>
#include <stdexcept>

namespace namb200
{

namespace
{

void add(std::vector<StateSegment>& segs, const std::string& name, int channels, long columns)
{
  if (columns <= 0)
    return;
  StateSegment s;
  s.name = name;
  s.channels = channels;
  s.columns = columns;
  s.offset = segs.empty() ? 0 : segs.back().offset + (long)segs.back().channels * segs.back().columns;
  segs.push_back(s);
}

void wavenet_segments(const WaveNetSpec& wn, const std::string& prefix, std::vector<StateSegment>& segs)
{
  for (size_t a = 0; a < wn.arrays.size(); a++)
  {
    const ArraySpec& A = wn.arrays[a];
    const std::string arr = prefix + "array" + std::to_string(a);
    for (size_t l = 0; l < A.layers.size(); l++)
      add(segs, arr + ".layer" + std::to_string(l) + ".conv", A.layers[l].conv.in, A.layers[l].conv.lookback());
    add(segs, arr + ".head", A.head_rechannel.in, A.head_rechannel.lookback());
  }
  if (wn.with_head)
    for (size_t i = 0; i < wn.post_head.convs.size(); i++)
      add(segs, prefix + "head.conv" + std::to_string(i), wn.post_head.convs[i].in, wn.post_head.convs[i].lookback());
  if (wn.condition_dsp)
    wavenet_segments(wn.condition_dsp->wavenet, prefix + "condition_dsp.", segs);
}

void generic_net_descs(const GNet& net, const GenericPlan& gp, std::vector<StateSegDesc>& out)
{
  auto conv = [&out](const GConv& v) {
    if (v.kernel <= 1)
      return;
    const int lb = (v.kernel - 1) * v.dilation;
    out.push_back(StateSegDesc{kSegRowRing, v.ring_off, v.in, v.in, lb, v.ring_mask, 0, lb * v.in});
  };
  for (int a = 0; a < net.n_arrays; a++)
  {
    const GArray& A = net.arrays[a];
    for (int l = 0; l < A.n_layers; l++)
      conv(gp.layers[(size_t)(A.layer0 + l)].conv);
    conv(A.head);
  }
  if (net.with_head)
    for (int i = 0; i < net.n_head_convs; i++)
      conv(net.head_convs[i]);
}

} // namespace

std::vector<StateSegment> state_segments(const ModelSpec& ms)
{
  std::vector<StateSegment> segs;
  switch (ms.arch)
  {
    case Arch::WaveNet: wavenet_segments(ms.wavenet, "", segs); break;
    case Arch::ConvNet:
      for (size_t i = 0; i < ms.convnet.blocks.size(); i++)
        add(segs, "block" + std::to_string(i) + ".conv", ms.convnet.blocks[i].conv.in, ms.convnet.blocks[i].conv.lookback());
      break;
    case Arch::LSTM:
      for (int l = 0; l < ms.lstm.num_layers; l++)
      {
        add(segs, "layer" + std::to_string(l) + ".h", ms.lstm.hidden, 1);
        add(segs, "layer" + std::to_string(l) + ".c", ms.lstm.hidden, 1);
      }
      break;
    case Arch::Linear: add(segs, "input", 1, (long)ms.linear.receptive_field - 1); break;
    default: break;
  }
  return segs;
}

long state_payload_floats(const std::vector<StateSegment>& segs)
{
  return segs.empty() ? 0 : segs.back().offset + (long)segs.back().channels * segs.back().columns;
}

StateRecordHeader state_record_header(const ModelSpec& ms, long payload_floats)
{
  StateRecordHeader h;
  std::memset(&h, 0, sizeof h);
  std::memcpy(h.magic, "NAMS", 4);
  h.version = kStateRecordVersion;
  h.architecture = (uint32_t)ms.arch;
  h.payload_floats = (uint64_t)payload_floats;
  h.fingerprint = ms.fingerprint;
  return h;
}

std::string state_layout_json(const ModelSpec& ms)
{
  const std::vector<StateSegment> segs = state_segments(ms);
  const long floats = state_payload_floats(segs);
  char buf[256];
  std::snprintf(buf, sizeof buf,
                "{\"architecture\": %d, \"header_bytes\": %d, \"payload_floats\": %ld, \"record_bytes\": %ld, "
                "\"fingerprint\": %" PRIu64 ", \"segments\": [",
                (int)ms.arch, kStateHeaderBytes, floats, kStateHeaderBytes + 4 * floats, ms.fingerprint);
  std::string s = buf;
  for (size_t i = 0; i < segs.size(); i++)
  {
    std::snprintf(buf, sizeof buf, "%s{\"name\": \"%s\", \"channels\": %d, \"columns\": %ld, \"offset\": %ld}", i ? ", " : "",
                  segs[i].name.c_str(), segs[i].channels, segs[i].columns, segs[i].offset);
    s += buf;
  }
  return s + "]}";
}

std::vector<StateSegDesc> state_descs(const ModelSpec& ms, const WaveNetPlan* plan, const GenericPlan* gplan)
{
  std::vector<StateSegDesc> d;
  if (ms.arch == Arch::WaveNet && plan)
  {
    for (int a = 0; a < plan->n_arrays; a++)
    {
      const ArrayDesc& A = plan->arrays[(size_t)a];
      const int cp = plan->cp[a], cr = plan->creal[a];
      for (int l = 0; l < A.n_layers; l++)
      {
        const LayerDesc& L = plan->layers[(size_t)(A.layer0 + l)];
        if (L.lookback > 0)
          d.push_back(StateSegDesc{kSegPlaneRing, L.ring_off, cp, cr, L.lookback, L.ring_mask, 0, L.lookback * cp / 4});
      }
      if (A.head_kernel > 1)
      {
        const int hl = (A.head_kernel - 1) * A.head_dilation;
        d.push_back(StateSegDesc{kSegPlaneRing, A.head_ring_off, cp, cr, hl, A.head_ring_mask, 0, hl * cp / 4});
      }
    }
  }
  else if (ms.arch == Arch::WaveNet && gplan)
  {
    generic_net_descs(gplan->net, *gplan, d);
    if (gplan->has_cond)
      generic_net_descs(gplan->cond, *gplan, d);
  }
  else if (ms.arch == Arch::ConvNet && gplan)
  {
    for (int i = 0; i < gplan->convnet.n_blocks; i++)
    {
      const GConv& v = gplan->convnet.convs[i];
      const int lb = (v.kernel - 1) * v.dilation;
      if (lb > 0)
        d.push_back(StateSegDesc{kSegRowRing, v.ring_off, v.in, v.in, lb, v.ring_mask, 0, lb * v.in});
    }
  }
  else if (ms.arch == Arch::LSTM)
  {
    // device state: per layer h[H] | c[H], the record's order
    const int n = ms.lstm.num_layers * 2 * ms.lstm.hidden;
    if (n > 0)
      d.push_back(StateSegDesc{kSegFlat, 0, 1, 1, n, 0, 0, n});
  }
  else if (ms.arch == Arch::Linear)
  {
    const int n = ms.linear.receptive_field - 1; // device state: the last rf-1 samples, oldest first
    if (n > 0)
      d.push_back(StateSegDesc{kSegFlat, 0, 1, 1, n, 0, 0, n});
  }
  else
    throw std::runtime_error("no per-stream state layout for this architecture");

  // the device segments must be the record's, one for one (LSTM: its segments as one flat run)
  const std::vector<StateSegment> segs = state_segments(ms);
  const long floats = state_payload_floats(segs);
  long canon = 0;
  for (StateSegDesc& s : d)
  {
    s.canon_off = (int)canon;
    canon += (long)s.lookback * s.cr;
  }
  const bool count_ok = ms.arch == Arch::LSTM ? (d.size() == (segs.empty() ? 0u : 1u)) : d.size() == segs.size();
  if (!count_ok || canon != floats)
    throw std::runtime_error("internal: device state layout (" + std::to_string(d.size()) + " segments, " + std::to_string(canon)
                             + " floats) does not match the state record (" + std::to_string(segs.size()) + " segments, "
                             + std::to_string(floats) + " floats)");
  if (ms.arch != Arch::LSTM)
    for (size_t i = 0; i < d.size(); i++)
      if (d[i].cr != segs[i].channels || d[i].lookback != segs[i].columns)
        throw std::runtime_error("internal: device state segment " + std::to_string(i) + " does not match " + segs[i].name);
  return d;
}

std::vector<StateChunk> state_chunks(const std::vector<StateSegDesc>& descs)
{
  std::vector<StateChunk> c;
  for (size_t s = 0; s < descs.size(); s++)
    for (int i = 0; i < descs[s].items; i += kStateThreads)
      c.push_back(StateChunk{(int)s, i});
  return c;
}

} // namespace namb200
