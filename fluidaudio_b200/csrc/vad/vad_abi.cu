// C ABI of voice activity detection (declared in include/fluidaudio_b200_vad.h) over vad_kernels.cu.  Every argument
// is checked here or in the session set before any copy or launch; every entry point that returns a status returns
// through guard() (c_abi.h), and the clip calls lease the pooled call context (call_context.h).
#include "../../../include/fluidaudio_b200_vad.h"
#include "../c_abi.h"
#include "vad.h"

#include <climits>
#include <cmath>
#include <memory>

struct fa_vad_stream {
    fa::vad::StreamSet set;
};

using namespace fa;
using namespace fa::vad;

namespace {

// Int(seconds * 16000.0) for a finite, non-negative duration whose count is below 2^62, so that 2 * count and every
// sample position plus or minus a count stay inside int64
bool samples_of(double seconds, long long *out) {
    const double x = seconds * 16000.0;
    if (!(x >= 0.0) || !(x < 4611686018427387904.0)) return false;   // NaN, negative, 2^62 or more, or +inf
    *out = (long long)x;
    return true;
}

int resolve(const fa_vad_config *c, Resolved &r, const char *where) {
    if (!c) return refuse("%s: cfg is NULL", where);
    if (!(c->min_speech_duration >= 0) || !(c->min_silence_duration >= 0) || !(c->max_speech_duration > 0) ||
        !(c->speech_padding >= 0) || !(c->min_silence_at_max_speech >= 0))
        return refuse("%s: durations must be >= 0 (max_speech_duration > 0), not NaN", where);
    if (!(c->silence_threshold_for_split >= 0 && c->silence_threshold_for_split <= 1))
        return refuse("%s: silence_threshold_for_split %g is outside [0, 1]", where, c->silence_threshold_for_split);
    if (!(c->negative_threshold_offset >= 0))
        return refuse("%s: negative_threshold_offset %g must be >= 0", where, c->negative_threshold_offset);
    if (c->has_negative_threshold && !(c->negative_threshold >= 0 && c->negative_threshold <= 1))
        return refuse("%s: negative_threshold %g is outside [0, 1]", where, c->negative_threshold);
    long long max_speech = 0;
    if (!samples_of(c->min_speech_duration, &r.min_speech) || !samples_of(c->min_silence_duration, &r.min_silence) ||
        !samples_of(c->speech_padding, &r.pad) || !samples_of(c->min_silence_at_max_speech, &r.min_silence_at_max) ||
        (!std::isinf(c->max_speech_duration) && !samples_of(c->max_speech_duration, &max_speech)))
        return refuse("%s: a duration is infinite or holds 2^62 samples or more", where);
    // Swift traps where Int(max * 16000) - 4096 - 2 * pad falls below INT64_MIN (a pad within 2^11 of 2^62)
    if (!std::isinf(c->max_speech_duration) && max_speech - kChunk < 0 &&
        2 * r.pad > LLONG_MAX + (max_speech - kChunk) + 1)
        return refuse("%s: Int(max_speech_duration * 16000) - 4096 - 2 * pad overflows int64", where);
    if (c->has_negative_threshold) {   // VadManager+Streaming.swift:46-50, VadTypes.swift:84-89
        r.threshold = swift_min(1.0f, c->negative_threshold + c->negative_threshold_offset);
        r.negative = c->negative_threshold;
    } else {
        r.threshold = c->default_threshold;
        r.negative = swift_max(r.threshold - c->negative_threshold_offset, 0.01f);
    }
    r.split = c->silence_threshold_for_split;
    r.use_max = c->use_max_possible_silence_at_max_speech ? 1 : 0;
    // max(0, Int(max * 16000) - 4096 - 2 * pad), formed without an intermediate outside int64
    r.max_speech = std::isinf(c->max_speech_duration) ? LLONG_MAX
                   : max_speech - kChunk > 2 * r.pad ? max_speech - kChunk - 2 * r.pad
                                                      : 0;
    return FA_OK;
}

bool offsets_ok(const int64_t *off, long long count) {
    if (!off || off[0] != 0) return false;
    for (long long i = 0; i < count; ++i)
        if (off[i + 1] < off[i] || off[i + 1] - off[i] > INT32_MAX || off[i + 1] > (1LL << 62)) return false;
    return true;
}

int clips_call(bool fsmn, bool on_device, const float *input, const int64_t *offsets, int32_t clips,
               const int64_t *total_samples, const fa_vad_config *cfg, int64_t *counts, int64_t *segments, size_t cap,
               int64_t *total) {
    const char *where = fsmn ? "fa_fsmn_vad_decide" : "fa_vad_segment";
    Resolved r{};
    if (!fsmn) {
        const int st = resolve(cfg, r, where);
        if (st != FA_OK) return st;
    }
    if (!total || clips < 0) return refuse("%s: total is NULL or clip_count %d < 0", where, clips);
    if (!offsets_ok(offsets, clips))
        return refuse("%s: offsets must be %lld offsets from 0, non-decreasing, each clip below 2^31 rows", where,
                      (long long)clips + 1);
    if (clips > 0 && (!counts || (!fsmn && !total_samples)))
        return refuse("%s: counts%s is NULL", where, fsmn ? "" : " or total_samples");
    if (offsets[clips] > 0 && !input) return refuse("%s: the input is NULL with %lld rows", where, (long long)offsets[clips]);
    if (cap > 0 && !segments) return refuse("%s: segments is NULL with capacity %lld", where, capacity(cap));
    if (!fsmn)
        for (int b = 0; b < clips; ++b)
            if (total_samples[b] > (1LL << 62))
                return refuse("%s: total_samples[%d] = %lld is beyond 2^62", where, b, (long long)total_samples[b]);
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) {
        return clip_call(C, fsmn, on_device, input, offsets, clips, total_samples, r, counts, segments, capacity(cap),
                         total);
    });
}

int stream_advance(fa_vad_stream *h, int32_t count, const int32_t *sessions, const float *probability,
                   const float *new_hidden, const float *new_cell, const fa_vad_config *cfg, bool device,
                   int64_t *events) {
    if (!h) return refuse("fa_vad_stream_advance: h is NULL");
    Resolved r{};
    const int st = resolve(cfg, r, "fa_vad_stream_advance");
    if (st != FA_OK) return st;
    return h->set.advance(count, sessions, probability, new_hidden, new_cell, r, device, events);
}

} // namespace

FA_API void fa_vad_default_config(fa_vad_config *cfg) {
    if (cfg) *cfg = fa_vad_config{0.85f, 0.15, 0.75, 14.0, 0.1, 0.3f, 0, 0.0f, 0.15f, 0.098, 1};
}

FA_API fa_status fa_vad_resolve(const fa_vad_config *cfg, fa_vad_resolved *out) {
    return guard(__func__, [&]() -> int {
        if (!out) return refuse("fa_vad_resolve: out is NULL");
        Resolved r{};
        const int st = resolve(cfg, r, "fa_vad_resolve");
        if (st != FA_OK) return st;
        *out = fa_vad_resolved{r.threshold,  r.negative,    r.split,      r.use_max,           r.min_speech,
                               r.min_silence, r.max_speech, r.pad,        r.min_silence_at_max};
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_vad_stream_create(fa_vad_stream **out) {
    return guard(__func__, [&]() -> int {
        if (!out) return refuse("fa_vad_stream_create: out is NULL");
        *out = nullptr;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        std::unique_ptr<fa_vad_stream> h(new fa_vad_stream());
        const int st = h->set.init();
        if (st != FA_OK) return st;
        *out = h.release();
        return FA_STATUS_OK;
    });
}

FA_API void fa_vad_stream_destroy(fa_vad_stream *h) { delete h; }

FA_API fa_status fa_vad_stream_open(fa_vad_stream *h, int32_t *session) {
    return guard(__func__, [&]() -> int {
        if (!h || !session) return refuse("fa_vad_stream_open: h or session is NULL");
        int id = -1;
        const int st = h->set.open(&id);
        if (st == FA_OK) *session = id;
        return st;
    });
}

FA_API fa_status fa_vad_stream_close(fa_vad_stream *h, int32_t session) {
    return guard(__func__, [&]() -> int { return h ? h->set.close(session) : refuse("fa_vad_stream_close: h is NULL"); });
}

FA_API fa_status fa_vad_stream_model_inputs(fa_vad_stream *h, int32_t count, const int32_t *sessions,
                                            const float *audio, const int64_t *offsets, float *audio_input,
                                            float *hidden, float *cell) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.model_inputs(count, sessions, audio, offsets, false, audio_input, hidden, cell)
                 : refuse("fa_vad_stream_model_inputs: h is NULL");
    });
}

FA_API fa_status fa_vad_stream_model_inputs_device(fa_vad_stream *h, int32_t count, const int32_t *sessions,
                                                   const float *d_audio, const int64_t *offsets,
                                                   float *d_audio_input, float *d_hidden, float *d_cell) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.model_inputs(count, sessions, d_audio, offsets, true, d_audio_input, d_hidden, d_cell)
                 : refuse("fa_vad_stream_model_inputs_device: h is NULL");
    });
}

FA_API fa_status fa_vad_stream_advance(fa_vad_stream *h, int32_t count, const int32_t *sessions,
                                       const float *probability, const float *new_hidden, const float *new_cell,
                                       const fa_vad_config *cfg, int64_t *events) {
    return guard(__func__, [&] {
        return stream_advance(h, count, sessions, probability, new_hidden, new_cell, cfg, false, events);
    });
}

FA_API fa_status fa_vad_stream_advance_device(fa_vad_stream *h, int32_t count, const int32_t *sessions,
                                              const float *d_probability, const float *d_new_hidden,
                                              const float *d_new_cell, const fa_vad_config *cfg,
                                              int64_t *d_events) {
    return guard(__func__, [&] {
        return stream_advance(h, count, sessions, d_probability, d_new_hidden, d_new_cell, cfg, true, d_events);
    });
}

FA_API fa_status fa_vad_stream_session_state(fa_vad_stream *h, int32_t session, fa_vad_stream_session_info *info,
                                             float *context, float *hidden, float *cell) {
    return guard(__func__, [&]() -> int {
        if (!h || !info) return refuse("fa_vad_stream_session_state: h or info is NULL");
        SessionInfo s{};
        const int st = h->set.state(session, &s, context, hidden, cell);
        if (st != FA_OK) return st;
        *info = fa_vad_stream_session_info{s.triggered, s.pending, s.temp_end, s.processed};
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_vad_segment(const float *probabilities, const int64_t *offsets, int32_t clip_count,
                                const int64_t *total_samples, const fa_vad_config *cfg, int64_t *counts,
                                int64_t *segments, size_t capacity, int64_t *total) {
    return guard(__func__, [&] {
        return clips_call(false, false, probabilities, offsets, clip_count, total_samples, cfg, counts, segments,
                          capacity, total);
    });
}

FA_API fa_status fa_vad_segment_device(const float *d_probabilities, const int64_t *offsets, int32_t clip_count,
                                       const int64_t *total_samples, const fa_vad_config *cfg, int64_t *counts,
                                       int64_t *d_segments, size_t capacity, int64_t *total) {
    return guard(__func__, [&] {
        return clips_call(false, true, d_probabilities, offsets, clip_count, total_samples, cfg, counts, d_segments,
                          capacity, total);
    });
}

FA_API fa_status fa_fsmn_vad_decide(const float *silence, const int64_t *offsets, int32_t clip_count,
                                    int64_t *counts, int64_t *segments, size_t capacity, int64_t *total) {
    return guard(__func__, [&] {
        return clips_call(true, false, silence, offsets, clip_count, nullptr, nullptr, counts, segments, capacity,
                          total);
    });
}

FA_API fa_status fa_fsmn_vad_decide_device(const float *d_silence, const int64_t *offsets, int32_t clip_count,
                                           int64_t *counts, int64_t *d_segments, size_t capacity, int64_t *total) {
    return guard(__func__, [&] {
        return clips_call(true, true, d_silence, offsets, clip_count, nullptr, nullptr, counts, d_segments, capacity,
                          total);
    });
}
