// NAM/get_dsp.h -- nam::get_dsp for the libnam_b200.so library (reference NAM/get_dsp.h:66-122).
#pragma once

#include <filesystem>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>

#include "dsp.h"

namespace nam
{

/// Thrown when a .nam file cannot be read / parsed / lacks a required key (reference NAM/nam_file.h:11-15)
class NamFileValidationError : public std::runtime_error
{
public:
  using std::runtime_error::runtime_error;
};

const std::string LATEST_FULLY_SUPPORTED_NAM_FILE_VERSION = "0.7.0";
const std::string EARLIEST_SUPPORTED_NAM_FILE_VERSION = "0.5.0";

struct DspLoadOptions
{
  /// std::nullopt = keep the thread's current prewarm-on-reset default; true/false override it for the
  /// model being loaded (reference NAM/get_dsp.h:70-78)
  std::optional<bool> prewarm = std::nullopt;
};

/// Load a .nam file.  Throws NamFileValidationError (file problems) or std::runtime_error (unsupported
/// version, unknown architecture, weight-count mismatch, an option the CUDA path does not implement, no
/// CUDA device) -- never returns nullptr.
std::unique_ptr<DSP> get_dsp(const std::filesystem::path config_filename, DspLoadOptions options = DspLoadOptions());

/// Same, also returning the parsed pieces of the file.
std::unique_ptr<DSP> get_dsp(const std::filesystem::path config_filename, dspData& returnedConfig,
                             DspLoadOptions options = DspLoadOptions());

/// From the JSON text of a .nam document (the reference's nlohmann::json overload, without the dependency).
std::unique_ptr<DSP> get_dsp_from_json_text(const std::string& nam_json_text, DspLoadOptions options = DspLoadOptions());

/// Library extension: a model carrying `batch` independent streams; use B200DSP::Handle() with
/// nam_b200_process_f32 for the batched entry point.
std::unique_ptr<DSP> get_dsp_batched(const std::filesystem::path config_filename, int batch,
                                     DspLoadOptions options = DspLoadOptions());

} // namespace nam
