// stream_state.h -- the per-stream state record: one stream's history in a format that does not depend on the kernel
// or geometry serving a handle (include/nam_b200.h: nam_b200_export_streams and friends).
//
// A record is a 64-byte header (StateRecordHeader) followed by float32 payload, little-endian.  The payload is the
// reference's own state in its own memory order:
//   WaveNet / ConvNet: one segment per convolution with a look-back (K-1)*d > 0 -- layer convolutions, A2-style head
//     convolutions, post-stack head convolutions; the main network first (layer arrays in order, each array's layers then
//     its head convolution, then the post-stack head), then a condition_dsp sub-model's segments in the same order.  A
//     segment holds the last look-back columns of that convolution's input, oldest first, each column the real channel
//     count contiguous (the column-major storage of the reference's RingBuffer).
//   LSTM: per layer h[H] then c[H].
//   Linear: the last receptive_field - 1 input samples, oldest first.
// Host code only declares here; the pack / unpack kernels are in stream_state.cuh.
#pragma once

#include <cstdint>
#include <string>
#include <vector>

#include "generic_pack.h"
#include "nam_model_spec.h"
#include "wavenet_pack.h"

namespace namb200
{

constexpr uint32_t kStateRecordVersion = 1;
constexpr int kStateHeaderBytes = 64;

struct StateRecordHeader
{
  char magic[4]; // "NAMS"
  uint32_t version; // kStateRecordVersion
  uint32_t architecture; // nam_b200_info.architecture of the model the record belongs to
  uint32_t reserved; // 0
  uint64_t payload_floats;
  uint64_t fingerprint; // ModelSpec::fingerprint
  uint8_t zero[32];
};
static_assert(sizeof(StateRecordHeader) == kStateHeaderBytes, "state record header is 64 bytes");

// one history buffer of the record
struct StateSegment
{
  std::string name;
  int channels = 0; // real channel count of a column
  long columns = 0;
  long offset = 0; // float offset in the payload
};

// The record's segments for a model (WaveNet, LSTM, Linear or ConvNet; a container has none of its own).
std::vector<StateSegment> state_segments(const ModelSpec& ms);
long state_payload_floats(const std::vector<StateSegment>& segs);
StateRecordHeader state_record_header(const ModelSpec& ms, long payload_floats);
// Host-only description of the record of a model: segments, record bytes, fingerprint (a small JSON object).
std::string state_layout_json(const ModelSpec& ms);

// ---- device side: where each segment lives in one stream's device state ----------------------------------------------
enum : int
{
  kSegPlaneRing = 0, // [Cp/4][R][4] rings of the fused / model-specialised / low-latency WaveNet kernels (pad channels 0)
  kSegRowRing = 1, // [R][C] rings of the general and ConvNet kernels
  kSegFlat = 2 // contiguous floats: LSTM h, c; the Linear history
};

struct StateSegDesc
{
  int kind;
  int dev_off; // float offset in the stream's device state
  int cp, cr; // padded and real channel counts (cp == cr except for plane rings)
  int lookback; // columns (flat: floats)
  int mask; // ring size - 1 (flat: unused)
  int canon_off; // float offset in the record payload
  int items; // work items: lookback * cp / 4 (plane), lookback * cr (row), lookback (flat)
};

// a block of the pack / unpack grid: kStateThreads consecutive items of one segment
struct StateChunk
{
  int seg, item0;
};

// one stream of a pack / unpack launch: StreamRef (jit_params.h); `alt` is read by pack only
static_assert(sizeof(StreamRef) == 16, "StreamRef is 16 bytes");

constexpr int kStateThreads = 256;

// The handle's descriptors in record order; exactly one of `plan` / `gplan` for WaveNet (fused / general kernel),
// gplan for ConvNet, neither for LSTM and Linear.  Throws if the layout does not match the record's segments.
std::vector<StateSegDesc> state_descs(const ModelSpec& ms, const WaveNetPlan* plan, const GenericPlan* gplan);
std::vector<StateChunk> state_chunks(const std::vector<StateSegDesc>& descs);

} // namespace namb200
