// Diarizer timelines in HBM (fa_diarizer_timeline_*): host bookkeeping (timeline_streams.cu) and the kernels' launchers
// (timeline_kernels.cu).  Arithmetic: timeline_core.cuh.
#pragma once

#include "fa_common.cuh"
#include "session_table.h"
#include "timeline_core.cuh"

namespace fa {
namespace timeline {

// The fields of fa_diarizer_timeline_config.
struct Config {
    int num_speakers;
    float frame_duration, onset, offset;
    int pad_on, pad_off, min_on, min_off, activity, max_stored;
    Params params() const { return Params{onset, offset, pad_on, pad_off, min_on, min_off, activity}; }
};

// create's checks; FA_INVALID_ARGUMENT with the error text set.
int check_config(const Config &c, int max_tentative_rows);

// Per-session descriptor of a push (one warp each).
struct PushJob {
    long long slot;               // the session's id: its scratch and rows
    long long cursor;             // finalized frames before the push
    long long n, m;               // finalized and tentative rows
    long long fin, ten;           // float offsets of its rows in the packed inputs
    long long stage;              // segment offset of its staging slots, `bound` segments per speaker
    long long bound;              // segment_bound(n, m)
    long long counts;             // index of its lane counts (session i: i * numSpeakers)
};

// Per-session descriptor of finalize (one CTA each): its m tentative rows go to the ring at the cursor.
struct FinalizeJob {
    long long slot, cursor, m;
};

// A session's host mirror.  The stored rows are the finalized frames [max(0, cursor - maxStoredFrames), cursor): frame
// f sits in ring row f % maxStoredFrames, so the ring's head and fill follow from the cursor.
struct TimelineSession {
    long long cursor;       // finalizedCursorFrame
    long long tentative;    // rows of tentativePredictions
};

struct Layout {
    int speakers;
    long long ring_rows, tentative_rows, slot_floats;   // per session: ring, then tentative rows, [rows x speakers]
};

int launch_push(const Config &c, const Layout &l, const PushJob *d_jobs, int count, const float *fin, const float *ten,
                StoredScratch *scratch, float *rows, Segment *stage, int *lane_counts, int64_t *fin_counts,
                int64_t *ten_counts, cudaStream_t s);
int launch_pack(const Layout &l, int lanes, const PushJob *d_jobs, const Segment *stage, const int *lane_counts,
                long long *lane_offsets, Segment *fin_out, Segment *ten_out, cudaStream_t s);
int launch_finalize(const Layout &l, const FinalizeJob *d_jobs, int count, float *rows, cudaStream_t s);

struct SessionInfo {
    long long finalized_frames, stored_frames, tentative_frames;
};

class TimelineSet {
  public:
    Config cfg{};

    int init(const Config &c, int max_tentative_rows);
    int open(int *session);
    int close(int session);
    int push(int count, const int *sessions, const float *fin, const int64_t *fin_rows, const float *ten,
             const int64_t *ten_rows, bool on_device, Segment *fin_out, long long fin_cap, Segment *ten_out,
             long long ten_cap, int64_t *fin_counts, int64_t *ten_counts);
    int finalize(int count, const int *sessions);
    int reset(int count, const int *sessions);
    int clear_speaker(int session, int speaker);
    int state(int session, SessionInfo *info, float *stored, float *tentative, Scratch *scratch);

  private:
    Layout layout{};
    Stream stream;
    SessionTable<TimelineSession> table;
    DeviceBuffer<StoredScratch> d_scratch;   // [slots x speakers]
    DeviceBuffer<float> d_rows;              // [slots x slot_floats]
    UploadStage<> push_desc, finalize_desc;
    DeviceBuffer<Segment> d_stage;
    DeviceBuffer<int> d_lane_counts;          // [2 x lanes]: finalized, tentative
    DeviceBuffer<long long> d_lane_offsets;   // [2 x lanes]
    DeviceBuffer<> staging;                   // the host variant's arrays (HostStaging, fa_common.cuh)
};

} // namespace timeline
} // namespace fa
