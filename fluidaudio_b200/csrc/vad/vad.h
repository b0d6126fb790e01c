// The host side of voice activity detection (vad_kernels.cu) behind the C ABI (vad_abi.cu): the Silero session set
// and the two clip calls.
#pragma once

#include "../call_context.h"
#include "../session_table.h"
#include "vad_core.cuh"

namespace fa {
namespace vad {

// Floats of a session slot: [context 64 | hidden 128 | cell 128 | pending context 64], and its int64 fields
constexpr int kSlotFloats = kContext + 2 * kState + kContext;
constexpr int kHiddenAt = kContext, kCellAt = kContext + kState, kPendingAt = kContext + 2 * kState;
enum : int { kProcessed = 0, kTriggered = 1, kTempEnd = 2, kPendingCount = 3, kSlotFields = 4 };

struct Mirror {
    bool pending = false;   // a staged chunk waits for its advance
};

struct SessionInfo {
    long long processed, temp_end;
    int triggered, pending;
};

class StreamSet {
  public:
    int init();
    int open(int *session);
    int close(int session);
    int model_inputs(int count, const int *sessions, const float *audio, const int64_t *offsets, bool device,
                     float *audio_input, float *hidden, float *cell);
    int advance(int count, const int *sessions, const float *probability, const float *new_hidden,
                const float *new_cell, const Resolved &r, bool device, int64_t *events);
    int state(int session, SessionInfo *info, float *context, float *hidden, float *cell);

  private:
    Stream stream;   // declared first, so destroyed last
    SessionTable<Mirror> table;
    DeviceBuffer<float> d_state;    // [slots x kSlotFloats]
    DeviceBuffer<long long> d_meta; // [slots x kSlotFields]
    UploadStage<> desc;             // the call's per-session descriptors
    DeviceBuffer<> d_io;            // device twins of a host-buffer call's arrays
};

// fa_vad_segment (fsmn false, r read) and fa_fsmn_vad_decide (fsmn true) on a call context
int clip_call(CallContext &C, bool fsmn, bool on_device, const float *input, const int64_t *offsets, int clips,
              const int64_t *total_samples, const Resolved &r, int64_t *counts, int64_t *segments, long long capacity,
              int64_t *total);

} // namespace vad
} // namespace fa
