// nam_model_spec.h -- host-side description of a .nam model: parsed config + weights
// unpacked into dense per-module tensors.  This is the product's own loader; it replaces
// (for the hot-path architectures) the reference's
//   NAM/nam_file.cpp:9-40            file validation
//   NAM/get_dsp.cpp:18-39,113-154    version gate, weights, sample rate, metadata
//   NAM/wavenet/model.cpp:913-1276   WaveNet config parser
//   NAM/wavenet/model.cpp:152-181,563-569,661-683  weight stream order
//   NAM/conv1d.cpp:11-56, NAM/dsp.cpp:363-398      Conv1D / Conv1x1 weight layouts
//   NAM/lstm.cpp:9-29,70-101,171-181 LSTM
//   NAM/linear.cpp:61-81,306-316     Linear
//   NAM/convnet.cpp:14-60,132-201,321-335  ConvNet
// No CUDA here: everything in this file runs once at load time on the host.
#pragma once

#include <cstdint>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <vector>

#include "json_lite.h"

namespace namb200
{

/// Same role as nam::NamFileValidationError (NAM/nam_file.h:11-15)
class NamFileValidationError : public std::runtime_error
{
public:
  using std::runtime_error::runtime_error;
};

enum class Arch
{
  WaveNet = 1,
  LSTM = 2,
  Linear = 3,
  Container = 4, // "SlimmableContainer": N complete sub-models, one active at a time (NAM/container.cpp)
  ConvNet = 5 // NAM/convnet.cpp: kernel-2 dilated Conv1D -> BatchNorm -> activation blocks, linear head
};

// Order of nam::activations::ActivationType (NAM/activations.h:26-39)
enum class ActType : int
{
  Tanh = 0,
  Hardtanh,
  Fasttanh,
  ReLU,
  LeakyReLU,
  PReLU,
  Sigmoid,
  SiLU,
  Hardswish,
  LeakyHardtanh,
  Softsign,
  Identity = 100
};

struct ActSpec
{
  ActType type = ActType::Identity;
  float slope = 0.01f; // LeakyReLU
  std::vector<float> slopes; // PReLU (1 entry = shared)
  float min_val = -1.0f, max_val = 1.0f, min_slope = 0.01f, max_slope = 0.01f; // LeakyHardtanh
};

enum class Gating : int
{
  None = 0,
  Gated = 1,
  Blended = 2
};

/// Dense 1x1 conv: y = W x (+ b); W is (out x in) row-major, block diagonal when grouped.
struct Conv1x1W
{
  int in = 0, out = 0, groups = 1;
  bool bias = false;
  std::vector<float> w, b;
};

/// Dense dilated conv: per tap k a (out x in) row-major matrix, tap 0 = oldest sample.
struct Conv1DW
{
  int in = 0, out = 0, kernel = 1, dilation = 1, groups = 1;
  bool bias = false;
  std::vector<float> w; // [k][o][i]
  std::vector<float> b;
  long lookback() const { return (long)(kernel - 1) * dilation; }
};

struct FilmSpec
{
  bool active = false, shift = false;
  int groups = 1;
  int dim = 0; // modulated dimension
  Conv1x1W css; // condition -> (shift ? 2 : 1) * dim, with bias
};

// FiLM sites in weight-stream order (NAM/wavenet/model.cpp:165-180)
enum FilmSite
{
  F_CONV_PRE = 0,
  F_CONV_POST,
  F_MIXIN_PRE,
  F_MIXIN_POST,
  F_ACT_PRE,
  F_ACT_POST,
  F_L1X1_POST,
  F_H1X1_POST,
  F_COUNT
};

struct LayerSpec
{
  Gating gating = Gating::None;
  ActSpec act, sec_act;
  Conv1DW conv; // channels -> (gated ? 2 : 1) * bottleneck, bias
  Conv1x1W mixin; // condition_size -> same, no bias
  bool has_l1x1 = true, has_h1x1 = false;
  Conv1x1W l1x1; // bottleneck -> channels, bias
  Conv1x1W h1x1; // bottleneck -> head1x1.out_channels, bias
  FilmSpec film[F_COUNT];
};

struct ArraySpec
{
  int input_size = 1, condition_size = 1, channels = 0, bottleneck = 0;
  int head_size = 0, head_kernel = 1, head_dilation = 1;
  bool head_bias = false;
  int groups_input = 1, groups_input_mixin = 1;
  bool l1x1_active = true;
  int l1x1_groups = 1;
  bool h1x1_active = false;
  int h1x1_out = 0, h1x1_groups = 1;
  Conv1x1W rechannel; // input_size -> channels, no bias
  std::vector<LayerSpec> layers;
  Conv1DW head_rechannel; // head_out_size -> head_size
  int head_out_size() const { return h1x1_active ? h1x1_out : bottleneck; }
  long receptive_field() const;
};

struct PostHeadSpec
{
  int in_channels = 0, channels = 0, out_channels = 0;
  ActSpec act;
  std::vector<Conv1DW> convs;
};

struct ModelSpec;

struct WaveNetSpec
{
  int in_channels = 1;
  std::vector<ArraySpec> arrays;
  bool with_head = false;
  PostHeadSpec post_head;
  float head_scale = 1.0f; // the LAST weight, not the JSON field (model.cpp:670)
  std::shared_ptr<ModelSpec> condition_dsp;
};

struct LstmCellW
{
  int input_size = 0, hidden = 0;
  std::vector<float> w; // (4H x (I+H)) row-major, gate rows i,f,g,o
  std::vector<float> b; // 4H
  std::vector<float> h0, c0; // trained initial state (lstm.cpp:24-28)
};

struct LstmSpec
{
  int num_layers = 0, input_size = 1, hidden = 0;
  std::vector<LstmCellW> cells;
  std::vector<float> head_w; // (out x H) row-major
  std::vector<float> head_b;
};

struct LinearSpec
{
  int receptive_field = 0;
  bool bias = false;
  std::vector<float> impulse; // as stored: impulse[0] multiplies the newest sample
  float bias_value = 0.0f;
};

/// NAM/convnet.cpp: a chain of blocks (kernel-2 dilated Conv1D, BatchNorm folded to y = x * scale + loc, activation)
/// and a linear head.
struct ConvNetSpec
{
  int channels = 0, groups = 1;
  bool batchnorm = false;
  struct Block
  {
    Conv1DW conv; // (first: in_channels) -> channels, kernel 2, bias iff no batchnorm (convnet.cpp:55-56)
    std::vector<float> scale, loc; // BatchNorm::BatchNorm (convnet.cpp:14-37), empty without batchnorm
  };
  std::vector<Block> blocks;
  ActSpec act;
  Conv1x1W head; // channels -> out_channels, bias (convnet.cpp:132-153)
};

struct ModelSpec
{
  Arch arch = Arch::WaveNet;
  std::string architecture; // as written in the file
  std::string version;
  double sample_rate = -1.0; // NAM_UNKNOWN_EXPECTED_SAMPLE_RATE
  int in_channels = 1, out_channels = 1;
  int prewarm_samples = 0; // DSP::GetPrewarmSamples()
  std::optional<double> loudness, input_level, output_level;
  size_t n_weights = 0;
  // FNV-1a 64 over the architecture name, the parsed "config" object (keys sorted, numbers as double bits) and the
  // float32 bits of the weights: the identity of a model's state layout and arithmetic, independent of load options
  // (fast_tanh) and of how the document was spelled.  Stamped into per-stream state records (stream_state.h).
  uint64_t fingerprint = 0;
  // the same hash without the weights and the config's unused "head_scale" field: equal for documents that differ only in
  // their weights (model banks, nam_b200_create_bank_from_json)
  uint64_t config_fingerprint = 0;
  WaveNetSpec wavenet;
  LstmSpec lstm;
  LinearSpec linear;
  ConvNetSpec convnet;
  // Arch::Container: (max_value, the sub-model's complete .nam document re-serialised); ascending max_value,
  // the last one >= 1.0 (ContainerModel ctor, container.cpp:19-47)
  struct Submodel
  {
    double max_value = 0.0;
    std::string model_json;
  };
  std::vector<Submodel> submodels;
};

enum class VersionSupport
{
  No = 0,
  Partial = 1,
  Yes = 2
};
VersionSupport version_support(const std::string& version);

struct LoadOptions
{
  /// Mirrors Activation::enable_fast_tanh() having been called before loading: every "Tanh"
  /// activation is replaced by the rational fast_tanh at construction (NAM/activations.cpp:168-177).
  bool fast_tanh = false;
};

/// Parse a whole .nam document (root object with version / architecture / config / weights).
ModelSpec model_spec_from_json(const json::Value& root, const LoadOptions& opts);
ModelSpec model_spec_from_text(const std::string& text, const LoadOptions& opts);
/// Read + validate a .nam file (throws NamFileValidationError like validate_nam_file()).
ModelSpec model_spec_from_file(const std::string& path, const LoadOptions& opts);

} // namespace namb200
