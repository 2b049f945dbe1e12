// NAM/dsp.h -- drop-in replacement for the reference header of the same path, for the inference hot
// path only: the nam::DSP interface (reference NAM/dsp.h:70-231) with the same public names, argument
// meaning and error behaviour, backed by libnam_b200.so (hand-written sm_90a kernels behind the C ABI
// of include/nam_b200.h) instead of Eigen.  No Eigen and no nlohmann types appear here, so a host that
// only uses the public DSP surface (the reference's tools/benchmodel.cpp, tools/render.cpp,
// tools/loadmodel.cpp, or the NeuralAmpModelerPlugin) compiles against it unchanged.
#pragma once

#include <atomic>
#include <filesystem>
#include <memory>
#include <string>
#include <vector>

#include "activations.h"

#ifdef NAM_SAMPLE_FLOAT
  #define NAM_SAMPLE float
#else
  #define NAM_SAMPLE double
#endif

#ifndef NAM_DEFAULT_MAX_BUFFER_SIZE
  #define NAM_DEFAULT_MAX_BUFFER_SIZE 4096
#endif

#define NAM_UNKNOWN_EXPECTED_SAMPLE_RATE -1.0

struct nam_b200_model; // opaque C-ABI handle

namespace nam
{

/// Thread-local default for "Reset() prewarms" of DSP objects constructed while it is alive
/// (reference NAM/dsp.h:44-57).
class ScopedPrewarmOnResetDefault
{
public:
  explicit ScopedPrewarmOnResetDefault(const bool prewarmOnReset);
  ~ScopedPrewarmOnResetDefault();
  ScopedPrewarmOnResetDefault(const ScopedPrewarmOnResetDefault&) = delete;
  ScopedPrewarmOnResetDefault& operator=(const ScopedPrewarmOnResetDefault&) = delete;
  bool PreviousPrewarmOnReset() const { return mPreviousPrewarmOnReset; }

private:
  bool mPreviousPrewarmOnReset;
};

/// Base class of all models.  The default process() copies input to output, exactly like the
/// reference's (NAM/dsp.cpp:103-119); models loaded by get_dsp() are subclasses backed by libnam_b200.so.
class DSP
{
public:
  DSP(const int in_channels, const int out_channels, const double expected_sample_rate);
  virtual ~DSP() = default;

  virtual void prewarm();
  /// input[channel][frame], output[channel][frame]; num_frames <= maxBufferSize of the last Reset()
  virtual void process(NAM_SAMPLE** input, NAM_SAMPLE** output, const int num_frames);

  double GetExpectedSampleRate() const { return mExpectedSampleRate; }
  int NumInputChannels() const { return mInChannels; }
  int NumOutputChannels() const { return mOutChannels; }
  double GetInputLevel();
  double GetLoudness() const; ///< throws std::runtime_error when unknown
  double GetOutputLevel();
  bool HasInputLevel();
  bool HasLoudness() const { return mHasLoudness; }
  bool HasOutputLevel();
  virtual int GetPrewarmSamples() { return 0; }
  virtual void Reset(const double sampleRate, const int maxBufferSize);
  void ResetAndPrewarm(const double sampleRate, const int maxBufferSize);
  virtual void SetPrewarmOnReset(const bool prewarmOnReset);
  bool GetPrewarmOnReset() const;
  void SetInputLevel(const double inputLevel);
  void SetLoudness(const double loudness);
  void SetOutputLevel(const double outputLevel);
  int GetMaxBufferSize() const { return mMaxBufferSize; }

protected:
  bool mHasLoudness = false;
  double mLoudness = 0.0;
  double mExpectedSampleRate;
  bool mHaveExternalSampleRate = false;
  double mExternalSampleRate = -1.0;
  int mMaxBufferSize = 0;
  std::atomic<bool> mPrewarmOnReset;

  virtual void SetMaxBufferSize(const int maxBufferSize);

private:
  const int mInChannels;
  const int mOutChannels;
  struct Level
  {
    bool haveLevel = false;
    float level = 0.0;
  };
  Level mInputLevel;
  Level mOutputLevel;
};

/// A model whose process() runs on the GPU (H100, sm_90a) through libnam_b200.so.  One object == one stream of the
/// handle (stream 0), so the reference's calling sequence get_dsp -> Reset -> process... works as is.
class B200DSP : public DSP
{
public:
  /// Takes ownership of the C-ABI handle.
  B200DSP(nam_b200_model* handle, const int in_channels, const int out_channels, const double expected_sample_rate,
          const int prewarm_samples);
  ~B200DSP() override;
  void prewarm() override;
  void process(NAM_SAMPLE** input, NAM_SAMPLE** output, const int num_frames) override;
  int GetPrewarmSamples() override { return mPrewarmSamples; }
  void Reset(const double sampleRate, const int maxBufferSize) override;
  nam_b200_model* Handle() { return mHandle; }

protected:
  nam_b200_model* mHandle;
  int mPrewarmSamples;
};

/// The pieces of a .nam file (reference NAM/dsp.h:348-357) with the JSON blocks kept as text, so this
/// header does not depend on a JSON library.
struct dspData
{
  std::string version;
  std::string architecture;
  std::string config; ///< JSON text of the "config" object
  std::string metadata; ///< JSON text of the "metadata" object ("null" when absent)
  std::vector<float> weights;
  double expected_sample_rate;
};

void verify_config_version(const std::string version);

} // namespace nam
