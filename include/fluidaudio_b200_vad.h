/* C ABI of voice activity detection in libfluidaudio_b200.so, beside the main header it builds on (status codes).
 * Plain C11, like the other headers under include/. */
#ifndef FLUIDAUDIO_B200_VAD_H
#define FLUIDAUDIO_B200_VAD_H

#include "fluidaudio_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Voice activity detection around the Silero and FSMN-VAD models (Sources/FluidAudio/VAD/): the models stay with the
 * caller, everything around them runs here for many sessions or clips per call.  Audio is 16 kHz mono float32.
 *
 * Silero geometry: a model step reads FA_VAD_MODEL_INPUT = FA_VAD_CONTEXT + FA_VAD_CHUNK samples (the session's
 * context, then the chunk) and an LSTM state of FA_VAD_STATE hidden and FA_VAD_STATE cell floats. */
#define FA_VAD_CHUNK 4096
#define FA_VAD_CONTEXT 64
#define FA_VAD_STATE 128
#define FA_VAD_MODEL_INPUT 4160

/* VadConfig.defaultThreshold and every field of VadSegmentationConfig (VadTypes.swift:4-91).  Durations are seconds. */
typedef struct {
    float default_threshold;                  /* 0.85 */
    double min_speech_duration;               /* 0.15 */
    double min_silence_duration;              /* 0.75 */
    double max_speech_duration;               /* 14.0; +inf: no split */
    double speech_padding;                    /* 0.1 */
    float silence_threshold_for_split;        /* 0.3 */
    int32_t has_negative_threshold;           /* 0: negative_threshold is nil */
    float negative_threshold;
    float negative_threshold_offset;          /* 0.15 */
    double min_silence_at_max_speech;         /* 0.098 */
    int32_t use_max_possible_silence_at_max_speech; /* 1 */
} fa_vad_config;

/* What a config resolves to.  threshold: min(1, negative + offset) in float32 with a negative threshold, else
 * default_threshold; negative_threshold: the override, else max(threshold - offset, 0.01f); sample counts are
 * Int(seconds * 16000.0), truncated in double; max_speech_samples is max(0, Int(max * 16000) - 4096 - 2 * pad), or
 * INT64_MAX when the duration is +inf.  min and max are Swift's (a NaN default threshold stays NaN). */
typedef struct {
    float threshold;
    float negative_threshold;
    float silence_threshold_for_split;
    int32_t use_max_possible_silence_at_max_speech;
    int64_t min_speech_samples;
    int64_t min_silence_samples;
    int64_t max_speech_samples;
    int64_t speech_pad_samples;
    int64_t min_silence_at_max_speech_samples;
} fa_vad_resolved;

/* Writes the reference defaults. */
void fa_vad_default_config(fa_vad_config *cfg);
/* Host only.  FA_STATUS_INVALID_ARGUMENT for what VadSegmentationConfig.init's preconditions trap on (a negative or
 * NaN duration, max_speech_duration <= 0, silence_threshold_for_split or a set negative_threshold outside [0, 1],
 * a negative or NaN offset), for a non-finite duration other than max_speech_duration = +inf, and for a duration whose
 * sample count is 2^62 or more (the sample arithmetic of both state machines then stays inside int64), or where
 * Int(max_speech_duration * 16000) - 4096 - 2 * pad falls below INT64_MIN, as Swift traps there.  The default
 * threshold is taken as given. */
fa_status fa_vad_resolve(const fa_vad_config *cfg, fa_vad_resolved *out);

/* Silero live sessions: VadManager.processStreamingChunk (VadManager+Streaming.swift) for many sessions, as two calls
 * around the caller's model.  A session holds VadStreamState (VadTypes.swift:93-219): context, hidden and cell state,
 * triggered, tempEndSample and processedSamples, in HBM.
 *
 * fa_vad_stream_model_inputs: session sessions[i] receives audio[offsets[i] .. offsets[i+1]) (count + 1
 * non-decreasing offsets, offsets[0] >= 0).  Row i of audio_input [count x 4160] is the session's context followed by
 * the chunk truncated to its first 4096 samples or padded to 4096 with its last sample (0 for an empty chunk); rows i
 * of hidden and cell [count x 128] are its LSTM state.  The call records a pending chunk per session (the last 64
 * samples of the processed chunk and the chunk's own sample count) and commits nothing; staging again before an
 * advance replaces it.
 *
 * fa_vad_stream_advance: the model's outputs for the same sessions (probability [count], new_hidden and new_cell
 * [count x 128]) commit each pending chunk: the pending context becomes the context, processedSamples grows by the
 * chunk's unpadded count, and streamingStateMachine (:31-91) runs with the resolved cfg.  events [count x 2] receives
 * per session (kind, sample index) as int64: kind 0 none (sample -1), 1 speech start, 2 speech end.  A NaN
 * probability takes neither branch.
 *
 * Both calls check every session first (open, no id twice, for advance a pending chunk each) and a refused call
 * changes nothing.  One launch each, none for count 0.  The host variants synchronise once; the _device variants take
 * every array but sessions and offsets in HBM and are asynchronous on the handle's stream.  Sessions are opened at
 * the lowest free id with VadStreamState.initial().  A handle is not thread-safe. */
typedef struct fa_vad_stream fa_vad_stream;

typedef struct {
    int32_t triggered;
    int32_t has_pending;
    int64_t temp_end_sample; /* -1: nil */
    int64_t processed_samples;
} fa_vad_stream_session_info;

fa_status fa_vad_stream_create(fa_vad_stream **out);
void fa_vad_stream_destroy(fa_vad_stream *h);
fa_status fa_vad_stream_open(fa_vad_stream *h, int32_t *session);
fa_status fa_vad_stream_close(fa_vad_stream *h, int32_t session);
fa_status fa_vad_stream_model_inputs(fa_vad_stream *h, int32_t count, const int32_t *sessions, const float *audio,
                                     const int64_t *offsets, float *audio_input, float *hidden, float *cell);
fa_status fa_vad_stream_model_inputs_device(fa_vad_stream *h, int32_t count, const int32_t *sessions,
                                            const float *d_audio, const int64_t *offsets, float *d_audio_input,
                                            float *d_hidden, float *d_cell);
fa_status fa_vad_stream_advance(fa_vad_stream *h, int32_t count, const int32_t *sessions, const float *probability,
                                const float *new_hidden, const float *new_cell, const fa_vad_config *cfg,
                                int64_t *events);
fa_status fa_vad_stream_advance_device(fa_vad_stream *h, int32_t count, const int32_t *sessions,
                                       const float *d_probability, const float *d_new_hidden,
                                       const float *d_new_cell, const fa_vad_config *cfg, int64_t *d_events);
/* The session's committed state; context [64], hidden [128] and cell [128] may each be NULL.  Synchronises. */
fa_status fa_vad_stream_session_state(fa_vad_stream *h, int32_t session, fa_vad_stream_session_info *info,
                                      float *context, float *hidden, float *cell);

/* Clip calls.  Clip b is rows offsets[b] .. offsets[b+1) of the input (clip_count + 1 non-decreasing offsets from 0,
 * each clip below 2^31 rows).  Outputs are (start, end) int64 pairs back to back in clip order: counts[b] pairs of
 * clip b, *total in all.  capacity (in pairs) below *total gives FA_STATUS_OUTPUT_TOO_SMALL with counts and *total set
 * and segments untouched.  Two launches (the per-clip state machine, the gather; the gather is skipped when *total is
 * 0 or the capacity short) and one synchronisation before the gather, on a pooled call context; a host-buffer call
 * also waits for its copy back.  The _device variants take the input and segments in HBM and return with the gather
 * queued.
 *
 * fa_vad_segment: segmentSpeech(from:totalSamples:config:) (VadManager+SpeechSegmentation.swift:22-51, 71-234) over
 * per-chunk Silero probabilities, total_samples[b] the clip's sample count: the speech sample ranges after the padding
 * pass and the final clamp and filter.  Chunk i starts at sample i * 4096 whatever total_samples is; total_samples
 * <= 0 or no probabilities gives no segments.
 *
 * fa_fsmn_vad_decide: FsmnVadManager.decide(silence:) (FsmnVadManager.swift:159-201) over per-frame silence
 * probabilities with the reference's fixed constants (10 ms frames): (startMs, endMs) per segment.  A NaN silence
 * probability is not speech. */
fa_status fa_vad_segment(const float *probabilities, const int64_t *offsets, int32_t clip_count,
                         const int64_t *total_samples, const fa_vad_config *cfg, int64_t *counts, int64_t *segments,
                         size_t capacity, int64_t *total);
fa_status fa_vad_segment_device(const float *d_probabilities, const int64_t *offsets, int32_t clip_count,
                                const int64_t *total_samples, const fa_vad_config *cfg, int64_t *counts,
                                int64_t *d_segments, size_t capacity, int64_t *total);
fa_status fa_fsmn_vad_decide(const float *silence, const int64_t *offsets, int32_t clip_count, int64_t *counts,
                             int64_t *segments, size_t capacity, int64_t *total);
fa_status fa_fsmn_vad_decide_device(const float *d_silence, const int64_t *offsets, int32_t clip_count,
                                    int64_t *counts, int64_t *d_segments, size_t capacity, int64_t *total);

#ifdef __cplusplus
}
#endif
#endif /* FLUIDAUDIO_B200_VAD_H */
