// C ABI of offline diarization's prepare stage (declared in include/fluidaudio_b200.h) over prepare_kernels.cu:
// segmentation windows and decoding, embedding windows and the embedding plan.  Every entry point that returns a status
// returns through guard() (c_abi.h), and the device calls lease the pooled call context.
#include "c_abi.h"
#include "call_context.h"
#include "prepare_plan.h"

#include <algorithm>
#include <climits>
#include <vector>

using namespace fa;

FA_API void fa_seg_default_config(fa_seg_config *cfg) {
    if (!cfg) return;
    const prepare::SegConfig d;
    cfg->sample_rate = d.sample_rate;
    cfg->speech_onset_threshold = d.speech_onset_threshold;
    cfg->window_duration = d.window_duration;
    cfg->step_ratio = d.step_ratio;
}

FA_API void fa_embed_plan_default_config(fa_embed_plan_config *cfg) {
    if (!cfg) return;
    const prepare::PlanConfig d;
    cfg->exclude_overlap = d.exclude_overlap ? 1 : 0;
    cfg->skip_threshold = d.skip_threshold;
    cfg->min_segment_duration = d.min_segment_duration;
    cfg->weight_frames = d.weight_frames;
    cfg->audio_sample_count = d.audio_sample_count;
    cfg->fbank_batch = d.fbank_batch;
    cfg->reserved = 0;
}

// The checked form of an fa_seg_config (OfflineDiarizerConfig.validate: window > 0, step ratio in (0, 1]).
static bool seg_config_of(const fa_seg_config *cfg, prepare::SegConfig &c) {
    if (!cfg) return false;
    c.sample_rate = cfg->sample_rate;
    c.window_duration = cfg->window_duration;
    c.step_ratio = cfg->step_ratio;
    c.speech_onset_threshold = cfg->speech_onset_threshold;
    if (prepare::seg_config_ok(c)) return true;
    fa::set_error("fa_seg_config: sample_rate and window_duration must be positive and step_ratio within (0, 1]");
    return false;
}

FA_API fa_status fa_seg_window_count(int64_t total_samples, const fa_seg_config *cfg, int32_t *chunks, int64_t *window,
                                     int64_t *step) {
    return guard(__func__, [&]() -> int {
        prepare::SegConfig c;
        if (total_samples < 0 || !seg_config_of(cfg, c)) return FA_STATUS_INVALID_ARGUMENT;
        const long long n = prepare::window_count(total_samples, c);
        if (n > INT32_MAX) return FA_STATUS_INDEX_OVERFLOW;
        if (chunks) *chunks = (int32_t)n;
        if (window) *window = prepare::samples_per_window(c);
        if (step) *step = prepare::samples_per_step(c);
        return FA_STATUS_OK;
    });
}

static int seg_windows(bool on_device, const float *audio, int64_t total_samples, const fa_seg_config *cfg,
                       int32_t first_chunk, int32_t chunk_count, float *out, double *chunk_offsets) {
    prepare::SegConfig c;
    if (total_samples < 0 || first_chunk < 0 || chunk_count < 0 || !seg_config_of(cfg, c)) return FA_STATUS_INVALID_ARGUMENT;
    if (total_samples == 0) {
        fa::set_error("noSpeechDetected: the audio holds no samples");
        return FA_STATUS_RUNTIME_ERROR;
    }
    if ((long long)first_chunk + chunk_count > prepare::window_count(total_samples, c))
        return refuse("fa_seg_windows: chunks %d .. %lld lie past the last window", first_chunk,
                      (long long)first_chunk + chunk_count - 1);
    if (chunk_count == 0) return FA_STATUS_OK;
    if (!audio || !out) return FA_STATUS_INVALID_ARGUMENT;
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    const long long window = prepare::samples_per_window(c), step = prepare::samples_per_step(c);
    std::vector<prepare::WindowDesc> desc((size_t)chunk_count);
    for (int32_t i = 0; i < chunk_count; ++i) {
        const long long offset = (long long)(first_chunk + i) * step;
        desc[i] = prepare::WindowDesc{offset, std::max(0LL, std::min(window, (long long)total_samples - offset))};
        if (chunk_offsets) chunk_offsets[i] = (double)offset / (double)c.sample_rate;
    }
    return with_context(0, [&](CallContext &C) {
        return prepare::gather_windows(C, on_device, audio, total_samples, desc.data(), chunk_count, window, out);
    });
}
FA_API fa_status fa_seg_windows(const float *audio, int64_t total_samples, const fa_seg_config *cfg, int32_t first_chunk,
                                int32_t chunk_count, float *out_windows, double *chunk_offsets) {
    return guard(__func__, [&] {
        return seg_windows(false, audio, total_samples, cfg, first_chunk, chunk_count, out_windows, chunk_offsets);
    });
}
FA_API fa_status fa_seg_windows_device(const float *d_audio, int64_t total_samples, const fa_seg_config *cfg,
                                       int32_t first_chunk, int32_t chunk_count, float *d_out_windows,
                                       double *chunk_offsets) {
    return guard(__func__, [&] {
        return seg_windows(true, d_audio, total_samples, cfg, first_chunk, chunk_count, d_out_windows, chunk_offsets);
    });
}

static int embed_windows(bool on_device, const float *audio, int64_t total_samples, const double *chunk_offsets,
                         int32_t offsets_count, const int32_t *chunk_index, int32_t count, const fa_seg_config *cfg,
                         int32_t audio_sample_count, float *out) {
    prepare::SegConfig c;
    if (total_samples < 0 || offsets_count < 0 || count < 0 || audio_sample_count < 1 || !seg_config_of(cfg, c) ||
        (offsets_count > 0 && !chunk_offsets))
        return FA_STATUS_INVALID_ARGUMENT;
    for (int32_t i = 0; chunk_index && i < count; ++i)
        if (chunk_index[i] < 0) return FA_STATUS_INVALID_ARGUMENT;
    if (count == 0) return FA_STATUS_OK;
    if (!out || (!audio && total_samples > 0)) return FA_STATUS_INVALID_ARGUMENT;
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    std::vector<prepare::WindowDesc> desc((size_t)count);
    for (int32_t i = 0; i < count; ++i) {
        const int chunk = chunk_index ? chunk_index[i] : i;
        desc[i] = prepare::embed_window(prepare::resolve_chunk_offset(chunk_offsets, offsets_count, chunk, c),
                                        total_samples, c, audio_sample_count);
    }
    return with_context(0, [&](CallContext &C) {
        return prepare::gather_windows(C, on_device, audio, total_samples, desc.data(), count, audio_sample_count, out);
    });
}
FA_API fa_status fa_embed_windows(const float *audio, int64_t total_samples, const double *chunk_offsets,
                                  int32_t offsets_count, const int32_t *chunk_index, int32_t count,
                                  const fa_seg_config *cfg, int32_t audio_sample_count, float *out) {
    return guard(__func__, [&] {
        return embed_windows(false, audio, total_samples, chunk_offsets, offsets_count, chunk_index, count, cfg,
                             audio_sample_count, out);
    });
}
FA_API fa_status fa_embed_windows_device(const float *d_audio, int64_t total_samples, const double *chunk_offsets,
                                         int32_t offsets_count, const int32_t *chunk_index, int32_t count,
                                         const fa_seg_config *cfg, int32_t audio_sample_count, float *d_out) {
    return guard(__func__, [&] {
        return embed_windows(true, d_audio, total_samples, chunk_offsets, offsets_count, chunk_index, count, cfg,
                             audio_sample_count, d_out);
    });
}

static int seg_decode(bool on_device, const float *logits, int32_t chunks, int32_t frames, int32_t classes,
                      const fa_seg_config *cfg, float *log_probs, float *speaker_weights, int64_t *histogram,
                      int64_t *speech_frames) {
    prepare::SegConfig c;
    if (chunks < 0 || frames < 0 || classes < 1 || classes > prepare::kMaxClasses || !seg_config_of(cfg, c))
        return FA_STATUS_INVALID_ARGUMENT;
    if (chunks == 0 || frames == 0) {
        for (int k = 0; histogram && k < 8; ++k) histogram[k] = 0;
        if (speech_frames) *speech_frames = 0;
        return FA_STATUS_OK;
    }
    if (!logits || !speaker_weights) return FA_STATUS_INVALID_ARGUMENT;
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) {
        return prepare::seg_decode(C, on_device, logits, chunks, frames, classes, c.speech_onset_threshold, log_probs,
                                   speaker_weights, histogram, speech_frames);
    });
}
FA_API fa_status fa_seg_decode(const float *logits, int32_t chunks, int32_t frames, int32_t classes,
                               const fa_seg_config *cfg, float *log_probs, float *speaker_weights, int64_t *class_histogram,
                               int64_t *speech_frames) {
    return guard(__func__, [&] {
        return seg_decode(false, logits, chunks, frames, classes, cfg, log_probs, speaker_weights, class_histogram,
                          speech_frames);
    });
}
FA_API fa_status fa_seg_decode_device(const float *d_logits, int32_t chunks, int32_t frames, int32_t classes,
                                      const fa_seg_config *cfg, float *d_log_probs, float *d_speaker_weights,
                                      int64_t *class_histogram, int64_t *speech_frames) {
    return guard(__func__, [&] {
        return seg_decode(true, d_logits, chunks, frames, classes, cfg, d_log_probs, d_speaker_weights, class_histogram,
                          speech_frames);
    });
}

static int embedding_plan(bool on_device, const float *weights, int32_t chunks, int32_t frames, int32_t speakers,
                          const double *chunk_offsets, int32_t offsets_count, double frame_duration,
                          int64_t total_samples, const fa_seg_config *seg_cfg, const fa_embed_plan_config *plan_cfg,
                          const prepare::PlanOutputs &out, int32_t *entry_count, int64_t *counters) {
    prepare::SegConfig c;
    if (chunks < 0 || frames < 0 || speakers < 0 || offsets_count < 0 || total_samples < 0 || !entry_count || !plan_cfg ||
        !seg_config_of(seg_cfg, c) || (offsets_count > 0 && !chunk_offsets))
        return FA_STATUS_INVALID_ARGUMENT;
    if (plan_cfg->weight_frames < 1 || plan_cfg->audio_sample_count < 1 || plan_cfg->fbank_batch < 1 ||
        !(plan_cfg->min_segment_duration >= 0.0))
        return refuse("fa_embed_plan_config: weight_frames, audio_sample_count and fbank_batch must be positive and "
                      "min_segment_duration >= 0");
    *entry_count = 0;
    for (int k = 0; counters && k < 4; ++k) counters[k] = 0;
    if (chunks == 0 || frames == 0 || speakers == 0) return FA_STATUS_OK;   // :655, :423-425
    if (!weights) return FA_STATUS_INVALID_ARGUMENT;
    if ((long long)chunks * speakers > INT32_MAX) return FA_STATUS_INDEX_OVERFLOW;
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    prepare::PlanConfig p;
    p.exclude_overlap = plan_cfg->exclude_overlap != 0;
    p.min_segment_duration = plan_cfg->min_segment_duration;
    p.skip_threshold = plan_cfg->skip_threshold;
    p.weight_frames = plan_cfg->weight_frames;
    p.audio_sample_count = plan_cfg->audio_sample_count;
    p.fbank_batch = plan_cfg->fbank_batch;
    return with_context(0, [&](CallContext &C) {
        return prepare::embedding_plan(C, on_device, weights, chunks, frames, speakers, chunk_offsets, offsets_count,
                                       frame_duration, total_samples, c, p, out, entry_count, counters);
    });
}
FA_API fa_status fa_embedding_plan(const float *speaker_weights, int32_t chunks, int32_t frames, int32_t speakers,
                                   const double *chunk_offsets, int32_t offsets_count, double frame_duration,
                                   int64_t total_samples, const fa_seg_config *seg_cfg,
                                   const fa_embed_plan_config *plan_cfg, int32_t *chunk_index, int32_t *speaker_index,
                                   int32_t *start_frame, int32_t *end_frame, double *start_time, double *end_time,
                                   float *mask_sum, int32_t *used_fallback, int32_t *reuse_of, float *frame_weights,
                                   float *model_weights, int32_t *entry_count, int64_t *counters) {
    return guard(__func__, [&] {
        const prepare::PlanOutputs out{chunk_index, speaker_index, start_frame, end_frame, start_time, end_time,
                                       mask_sum, used_fallback, reuse_of, frame_weights, model_weights};
        return embedding_plan(false, speaker_weights, chunks, frames, speakers, chunk_offsets, offsets_count,
                              frame_duration, total_samples, seg_cfg, plan_cfg, out, entry_count, counters);
    });
}
FA_API fa_status fa_embedding_plan_device(const float *d_speaker_weights, int32_t chunks, int32_t frames, int32_t speakers,
                                          const double *chunk_offsets, int32_t offsets_count, double frame_duration,
                                          int64_t total_samples, const fa_seg_config *seg_cfg,
                                          const fa_embed_plan_config *plan_cfg, int32_t *d_chunk_index,
                                          int32_t *d_speaker_index, int32_t *d_start_frame, int32_t *d_end_frame,
                                          double *d_start_time, double *d_end_time, float *d_mask_sum,
                                          int32_t *d_used_fallback, int32_t *d_reuse_of, float *d_frame_weights,
                                          float *d_model_weights, int32_t *entry_count, int64_t *counters) {
    return guard(__func__, [&] {
        const prepare::PlanOutputs out{d_chunk_index, d_speaker_index, d_start_frame, d_end_frame, d_start_time,
                                       d_end_time,    d_mask_sum,      d_used_fallback, d_reuse_of, d_frame_weights,
                                       d_model_weights};
        return embedding_plan(true, d_speaker_weights, chunks, frames, speakers, chunk_offsets, offsets_count,
                              frame_duration, total_samples, seg_cfg, plan_cfg, out, entry_count, counters);
    });
}

FA_API fa_status fa_weight_resample(const float *rows, int64_t row_count, int32_t in_len, int32_t out_len, float *out) {
    return guard(__func__, [&]() -> int {
        if (row_count < 0 || in_len < 1 || out_len < 1) return FA_STATUS_INVALID_ARGUMENT;
        if (row_count == 0) return FA_STATUS_OK;
        if (!rows || !out) return FA_STATUS_INVALID_ARGUMENT;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) {
            return prepare::weight_resample(C, rows, row_count, in_len, out_len, out);
        });
    });
}
