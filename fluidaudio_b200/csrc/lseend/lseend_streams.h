// The session set behind fa_lseend_stream_* (lseend_streams.cu): LSEENDFeatureProvider for many live sessions on one
// mel plan, their queues and running means in HBM, their lengths on the host (lseend_plan.h).
#pragma once

#include "lseend_plan.h"
#include "mel_plan.h"
#include "session_table.h"

namespace fa {
namespace lseend {

struct SessionInfo {
    long long audio_samples, mel_rows, cmn_count;
    int decoder_mask_end, has_snapshot;
};

class StreamSet {
  public:
    int init(const Config &c);
    int open(int *session);
    int close(int session);
    // chunks the next push of n samples (drain 0/1) to `session` emits; -1 for a closed session or n < 0
    long long chunks(int session, long long n, bool drain) const;
    // Session sessions[i] receives audio[offsets[i] .. offsets[i+1]), then the silence drain when drain[i] != 0, then
    // emits every ready chunk.  Outputs in call order: features [chunks x mel_frames x n_mels], masks [chunks x
    // chunk_size], warm-up counts [chunks]; chunks[i] receives session i's count.  device: audio and the three outputs
    // are HBM and the call is asynchronous on the set's stream.
    int push(int count, const int *sessions, const float *audio, const int64_t *offsets, const int *drain, bool device,
             float *features, long long features_len, float *masks, long long masks_len, int *warmup,
             long long warmup_len, int64_t *chunks);
    int snapshot(int count, const int *sessions);
    int rollback(int count, const int *sessions);
    int reset(int count, const int *sessions);
    int state(int session, SessionInfo *info, float *audio, float *mel, float *cmn_mean);

    const Sizes &sizes() const { return sz; }
    mel::MelPlan plan;   // the provider's AudioMelSpectrogram (:70-81); its compute stream is the set's stream

  private:
    int slots(int kind, int count, const int *sessions, const char *where);

    Config cfg{};
    Sizes sz{};
    int half = 0;      // floats of one half of a slot: [audio carry | mel rows], 16-byte aligned parts
    int mel_off = 0;   // offset of the mel rows inside a half
    int mean_half = 0; // floats of one half of a mean slot
    SessionTable<Session> table;
    DeviceBuffer<float> d_state;   // [slots x 2 x half]: live, then snapshot
    DeviceBuffer<float> d_mean;    // [slots x 2 x mean_half]: cmnMean, live then snapshot
    UploadStage<> desc;            // jobs and units of a push, session ids of a snapshot / rollback / reset
    DeviceBuffer<float> d_arena;   // every emitting session's audio input and mel queue of a push
};

} // namespace lseend
} // namespace fa
