// The host side of streaming speaker tracking (online_diar_kernels.cu) behind the C ABI (online_diar_abi.cu): the
// session set with its speaker databases in HBM, and the two handle-less model-input calls.
#pragma once

#include "../call_context.h"
#include "../session_table.h"
#include "online_diar_core.cuh"

#include <vector>

namespace fa {
namespace od {

struct Mirror {
    bool pending = false;   // embedding inputs staged a chunk that waits for its advance
    SessionMeta meta{};     // the device header, exact after every call
};

// A speaker as the ABI reads and writes it (fa_od_speaker)
struct SpeakerView {
    long long key, numeric, update_count;
    float duration;
    int named, has_numeric, permanent, raw_count;
};

class Databases {
  public:
    int init(int frames);
    int frames() const { return frames_; }
    int open(int *session);
    int close(int session);
    int embedding_inputs(int count, const int *sessions, const float *logits, long long chunk_size,
                         const Resolved &r, bool device, float *masks, int32_t *need);
    int advance(int count, const int *sessions, const float *embeddings, const double *offsets, const Resolved &r,
                bool device, int64_t *assigned, int32_t *seg_counts, int64_t *seg_ids, float *seg_values);
    int query(int session, int count, const float *embeddings, bool device, float *distances);
    int speaker_count(int session, long long *count, long long *next_id);
    int read(int session, SpeakerView *views, float *current, float *raws);
    // Replaces one session's database with `db` (the database operations run on a host copy, then land here)
    int load(int session, std::vector<Speaker> &db);
    int write(int session, const std::vector<Speaker> &db, const SessionMeta &meta);
    long long next_seq(long long n) {
        const long long s = seq_;
        seq_ += n;
        return s;
    }

  private:
    int reserve(int need_speakers);
    int grow(int slots, int capacity);
    Stream stream;   // declared first, so destroyed last
    SessionTable<Mirror> table;
    int frames_ = 0, capacity_ = 0;   // speakers per session slot
    long long seq_ = 0;               // the raw embeddings' sequence numbers
    DeviceBuffer<Speaker> d_db;       // [slots x capacity_]
    DeviceBuffer<SessionMeta> d_meta; // [slots]
    DeviceBuffer<unsigned char> d_bits; // [slots x (frames + 1)]: binarized frames, then the need bits
    UploadStage<> desc;
    DeviceBuffer<> d_io;
    PinnedBuffer<SessionMeta> h_meta;
};

// fa_od_chunk_inputs (chunk_size > 0, mask null) and fa_od_enrollment_inputs (chunk_size 0: each clip is its own
// length, segmentation null, a mask row of `frames` per clip)
int inputs_call(CallContext &C, bool on_device, const float *audio, const int64_t *offsets, int count,
                long long chunk_size, float *segmentation, float *waveform, float *mask, int frames);

} // namespace od
} // namespace fa
