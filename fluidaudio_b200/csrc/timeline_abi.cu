// C ABI of the diarizer timelines (declared in include/fluidaudio_b200.h): DiarizerTimeline's numeric core for many
// sessions in HBM, timeline_streams.cu and timeline_kernels.cu.  Every entry point that returns a status returns
// through guard() (c_abi.h).
#include "c_abi.h"
#include "timeline_plan.h"

#include <cmath>
#include <cstddef>
#include <memory>

struct fa_diarizer_timeline {
    fa::timeline::TimelineSet set;
};

using namespace fa;

#define FA_SAME_FIELD(a, b) (offsetof(timeline::Scratch, a) == offsetof(fa_diarizer_timeline_scratch, b))
static_assert(sizeof(timeline::Scratch) == sizeof(fa_diarizer_timeline_scratch) && FA_SAME_FIELD(start, start_frame) &&
                  FA_SAME_FIELD(end, end_frame) && FA_SAME_FIELD(unmerged_start, unmerged_start_frame) &&
                  FA_SAME_FIELD(count, active_frame_count) &&
                  FA_SAME_FIELD(unmerged_count, unmerged_active_frame_count) && FA_SAME_FIELD(sum, activity_sum) &&
                  FA_SAME_FIELD(unmerged_sum, unmerged_activity_sum) && FA_SAME_FIELD(speaking, speaking) &&
                  FA_SAME_FIELD(has_segment, has_segment),
              "timeline::Scratch is laid out as fa_diarizer_timeline_scratch");
#undef FA_SAME_FIELD

static timeline::Config timeline_config_of(const fa_diarizer_timeline_config *c) {
    return timeline::Config{c->num_speakers,     c->frame_duration_seconds, c->onset_threshold, c->offset_threshold,
                            c->onset_pad_frames, c->offset_pad_frames,      c->min_frames_on,   c->min_frames_off,
                            c->activity_type,    c->max_stored_frames};
}

FA_API fa_status fa_diarizer_timeline_default_config(fa_diarizer_timeline_config *cfg, int32_t preset,
                                                     int32_t num_speakers, float frame_duration_seconds) {
    return guard(__func__, [&]() -> int {
        if (!cfg) return FA_STATUS_INVALID_ARGUMENT;
        // DiarizerTimelineConfig.default(numSpeakers:frameDurationSeconds:) and sortformerDefault (:72-87)
        if (preset == FA_TIMELINE_PRESET_SORTFORMER) {
            num_speakers = 4;
            frame_duration_seconds = 0.08f;
        } else if (preset != FA_TIMELINE_PRESET_DEFAULT) {
            return refuse("fa_diarizer_timeline_default_config: unknown preset %d", preset);
        }
        *cfg = fa_diarizer_timeline_config{num_speakers, frame_duration_seconds, 0.5f, 0.5f, 0, 0, 0, 0,
                                           FA_TIMELINE_SIGMOIDS, FA_TIMELINE_DEFAULT_STORED_FRAMES};
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_diarizer_timeline_config_from_seconds(fa_diarizer_timeline_config *cfg, float onset_pad_seconds,
                                                          float offset_pad_seconds, float min_duration_on,
                                                          float min_duration_off) {
    return guard(__func__, [&]() -> int {
        if (!cfg) return FA_STATUS_INVALID_ARGUMENT;
        // Int(round(seconds / frameDurationSeconds)) in Float (:156-159); Swift's round is roundf, half away from zero
        const float secs[4] = {onset_pad_seconds, offset_pad_seconds, min_duration_on, min_duration_off};
        int32_t frames[4];
        for (int k = 0; k < 4; ++k) {
            const float r = roundf(secs[k] / cfg->frame_duration_seconds);
            if (!(r >= -2147483648.0f && r < 2147483648.0f))
                return refuse("fa_diarizer_timeline_config_from_seconds: %g s / %g s is not a finite int32 frame count",
                              (double)secs[k], (double)cfg->frame_duration_seconds);
            frames[k] = (int32_t)r;
        }
        cfg->onset_pad_frames = frames[0];
        cfg->offset_pad_frames = frames[1];
        cfg->min_frames_on = frames[2];
        cfg->min_frames_off = frames[3];
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_diarizer_timeline_segment_bound(int32_t num_speakers, int32_t count, const int64_t *finalized_rows,
                                                    const int64_t *tentative_rows, int64_t *finalized_bound,
                                                    int64_t *tentative_bound) {
    return guard(__func__, [&]() -> int {
        if (num_speakers < 1 || count < 0 || (count > 0 && (!finalized_rows || !tentative_rows)) || !finalized_bound ||
            !tentative_bound)
            return FA_STATUS_INVALID_ARGUMENT;
        int64_t f = 0, t = 0;
        for (int32_t i = 0; i < count; ++i) {
            if (finalized_rows[i] < 0 || tentative_rows[i] < 0) return FA_STATUS_INVALID_ARGUMENT;
            f += num_speakers * timeline::finalized_bound(finalized_rows[i]);
            t += num_speakers * timeline::tentative_bound(tentative_rows[i]);
        }
        *finalized_bound = f;
        *tentative_bound = t;
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_diarizer_timeline_create(const fa_diarizer_timeline_config *cfg, int32_t max_tentative_rows,
                                             fa_diarizer_timeline **out) {
    return guard(__func__, [&]() -> int {
        if (!cfg || !out) return FA_STATUS_INVALID_ARGUMENT;
        *out = nullptr;
        const timeline::Config c = timeline_config_of(cfg);
        int st = timeline::check_config(c, max_tentative_rows);
        if (st != FA_OK) return st;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        std::unique_ptr<fa_diarizer_timeline> h(new fa_diarizer_timeline());
        st = h->set.init(c, max_tentative_rows);
        if (st != FA_OK) return st;
        *out = h.release();
        return FA_STATUS_OK;
    });
}

FA_API void fa_diarizer_timeline_destroy(fa_diarizer_timeline *h) { delete h; }

FA_API fa_status fa_diarizer_timeline_open(fa_diarizer_timeline *h, int32_t *session) {
    return guard(__func__, [&]() -> int {
        if (!h || !session) return FA_STATUS_INVALID_ARGUMENT;
        int id = -1;
        const int st = h->set.open(&id);
        if (st == FA_OK) *session = id;
        return st;
    });
}

FA_API fa_status fa_diarizer_timeline_close(fa_diarizer_timeline *h, int32_t session) {
    return guard(__func__, [&]() -> int {
        if (!h) return FA_STATUS_INVALID_ARGUMENT;
        return h->set.close(session);
    });
}

static int timeline_push(fa_diarizer_timeline *h, int32_t count, const int32_t *sessions, const float *fin,
                         const int64_t *fin_rows, const float *ten, const int64_t *ten_rows, bool device,
                         fa_diarizer_timeline_segment *fin_out, size_t fin_cap, fa_diarizer_timeline_segment *ten_out,
                         size_t ten_cap, int64_t *fin_counts, int64_t *ten_counts) {
    if (!h) return FA_STATUS_INVALID_ARGUMENT;
    return h->set.push(count, sessions, fin, fin_rows, ten, ten_rows, device, fin_out, capacity(fin_cap), ten_out,
                       capacity(ten_cap), fin_counts, ten_counts);
}

FA_API fa_status fa_diarizer_timeline_push(fa_diarizer_timeline *h, int32_t count, const int32_t *sessions,
                                           const float *finalized, const int64_t *finalized_rows, const float *tentative,
                                           const int64_t *tentative_rows,
                                           fa_diarizer_timeline_segment *finalized_segments, size_t finalized_capacity,
                                           fa_diarizer_timeline_segment *tentative_segments, size_t tentative_capacity,
                                           int64_t *finalized_counts, int64_t *tentative_counts) {
    return guard(__func__, [&] {
        return timeline_push(h, count, sessions, finalized, finalized_rows, tentative, tentative_rows, false,
                             finalized_segments, finalized_capacity, tentative_segments, tentative_capacity,
                             finalized_counts, tentative_counts);
    });
}

FA_API fa_status fa_diarizer_timeline_push_device(fa_diarizer_timeline *h, int32_t count, const int32_t *sessions,
                                                  const float *d_finalized, const int64_t *finalized_rows,
                                                  const float *d_tentative, const int64_t *tentative_rows,
                                                  fa_diarizer_timeline_segment *d_finalized_segments,
                                                  size_t finalized_capacity,
                                                  fa_diarizer_timeline_segment *d_tentative_segments,
                                                  size_t tentative_capacity, int64_t *d_finalized_counts,
                                                  int64_t *d_tentative_counts) {
    return guard(__func__, [&] {
        return timeline_push(h, count, sessions, d_finalized, finalized_rows, d_tentative, tentative_rows, true,
                             d_finalized_segments, finalized_capacity, d_tentative_segments, tentative_capacity,
                             d_finalized_counts, d_tentative_counts);
    });
}

FA_API fa_status fa_diarizer_timeline_finalize(fa_diarizer_timeline *h, int32_t count, const int32_t *sessions) {
    return guard(__func__, [&]() -> int {
        if (!h) return FA_STATUS_INVALID_ARGUMENT;
        return h->set.finalize(count, sessions);
    });
}

FA_API fa_status fa_diarizer_timeline_reset(fa_diarizer_timeline *h, int32_t count, const int32_t *sessions) {
    return guard(__func__, [&]() -> int {
        if (!h) return FA_STATUS_INVALID_ARGUMENT;
        return h->set.reset(count, sessions);
    });
}

FA_API fa_status fa_diarizer_timeline_clear_speaker(fa_diarizer_timeline *h, int32_t session, int32_t speaker) {
    return guard(__func__, [&]() -> int {
        if (!h) return FA_STATUS_INVALID_ARGUMENT;
        return h->set.clear_speaker(session, speaker);
    });
}

FA_API fa_status fa_diarizer_timeline_session_state(fa_diarizer_timeline *h, int32_t session,
                                                    fa_diarizer_timeline_session_info *info, float *stored,
                                                    float *tentative, fa_diarizer_timeline_scratch *scratch) {
    return guard(__func__, [&]() -> int {
        if (!h || !info) return FA_STATUS_INVALID_ARGUMENT;
        timeline::SessionInfo s;
        const int st = h->set.state(session, &s, stored, tentative, reinterpret_cast<timeline::Scratch *>(scratch));
        if (st != FA_OK) return st;
        *info = fa_diarizer_timeline_session_info{s.finalized_frames, s.stored_frames, s.tentative_frames};
        return FA_STATUS_OK;
    });
}
