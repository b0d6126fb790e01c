/* C ABI of streaming speaker tracking in libfluidaudio_b200.so, beside the main header it builds on (status codes).
 * Plain C11, like the other headers under include/. */
#ifndef FLUIDAUDIO_B200_ONLINE_DIAR_H
#define FLUIDAUDIO_B200_ONLINE_DIAR_H

#include "fluidaudio_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* DiarizerManager's streaming diarization and SpeakerManager's speaker database (Sources/FluidAudio/Diarizer/Core,
 * Clustering, Segmentation, Extraction) for many live sessions per call.  The pyannote segmentation model and the
 * WeSpeaker embedding model stay with the caller; a chunk is three calls around them:
 *   fa_od_chunk_inputs       the segmentation model's waveform and the embedding model's (row 0 of its [3, 160000])
 *   fa_od_embedding_inputs   after the segmentation model: each local speaker's mask row (row 0 of [3, F]) and
 *                            whether the embedding model runs for it
 *   fa_od_advance            after the embedding model: speaker assignment into each session's database, then the
 *                            chunk's segments
 * Audio is 16 kHz mono float32.  F is the segmentation model's frame count per chunk (589 for the shipped model). */
#define FA_OD_DIM 256             /* embedding size */
#define FA_OD_FIFO 50             /* raw embeddings kept per speaker */
#define FA_OD_CLASSES 7           /* powerset classes per frame */
#define FA_OD_LOCAL 3             /* local speakers per chunk */
#define FA_OD_MODEL_SAMPLES 160000

/* DiarizerConfig (DiarizerTypes.swift).  min_embedding_update_duration, min_silence_gap and num_clusters are carried
 * for completeness: DiarizerManager does not read them. */
typedef struct {
    float clustering_threshold;          /* 0.7 */
    float min_speech_duration;           /* 1.0 */
    float min_embedding_update_duration; /* 2.0 */
    float min_silence_gap;               /* 0.5 */
    int32_t num_clusters;                /* -1 */
    float min_active_frames_count;       /* 10.0 */
    float chunk_duration;                /* 10.0 */
    float chunk_overlap;                 /* 0.0 */
} fa_od_config;

/* What a config resolves to: the thresholds in float32 (clustering_threshold * 1.2f and * 0.8f), and
 * chunk_size = 16000 * Int(chunk_duration.rounded()), step_size = chunk_size - 16000 * Int(chunk_overlap.rounded()),
 * rounding half away from zero.  A step of 0 or less yields no chunks. */
typedef struct {
    float speaker_threshold;
    float embedding_threshold;
    float min_speech_duration;
    float min_active_frames_count;
    int64_t chunk_size;
    int64_t step_size;
} fa_od_resolved;

/* One speaker of a database.  Identity is (named, key): named 0 is the canonical decimal id `key` (what
 * String(Int) writes, as every speaker the tracker creates has); named 1 is any other string, which the caller maps
 * to a key of its choosing.  numeric is Int(id) when has_numeric.  raw_count raw embeddings follow, oldest first. */
typedef struct {
    int64_t key;
    int64_t numeric;
    int64_t update_count;
    float duration;
    int32_t named;
    int32_t has_numeric;
    int32_t permanent;
    int32_t raw_count;
} fa_od_speaker;

/* SpeakerInitializationMode */
#define FA_OD_MODE_RESET 0
#define FA_OD_MODE_MERGE 1
#define FA_OD_MODE_OVERWRITE 2
#define FA_OD_MODE_SKIP 3

typedef struct fa_od_databases fa_od_databases;

/* Writes the reference defaults. */
void fa_od_default_config(fa_od_config *cfg);
/* Host only.  FA_STATUS_INVALID_ARGUMENT where Swift traps: a chunk duration or overlap that is not finite or whose
 * rounded value times 16000 leaves int64, a chunk size of 0 or less (its buffer cannot be made), a step of 0. */
fa_status fa_od_resolve(const fa_od_config *cfg, fa_od_resolved *out);

/* Model inputs for `count` chunks (samples offsets[b] .. offsets[b + 1] of `audio`, offsets from 0 and
 * non-decreasing): each chunk's first min(length, chunk_size) samples zero-padded to chunk_size and then truncated or
 * zero-filled to 160000 (segmentation, [count x 160000]), and the same chunk repeat-padded to 160000 samples, period
 * chunk_size (waveform, [count x 160000]).  One launch. */
fa_status fa_od_chunk_inputs(const float *audio, const int64_t *offsets, int32_t count, int64_t chunk_size,
                             float *segmentation, float *waveform);
fa_status fa_od_chunk_inputs_device(const float *d_audio, const int64_t *offsets, int32_t count, int64_t chunk_size,
                                    float *d_segmentation, float *d_waveform);
/* extractSpeakerEmbedding(from:)'s inputs for `count` clips: each clip repeat-padded (or truncated) to 160000 samples
 * (waveform, [count x 160000]; zeros for an empty clip) and its all-ones mask of `frames` entries (mask,
 * [count x frames]; zeros where numMasksInChunk is 0).  One launch. */
fa_status fa_od_enrollment_inputs(const float *audio, const int64_t *offsets, int32_t count, int32_t frames,
                                  float *waveform, float *mask);
fa_status fa_od_enrollment_inputs_device(const float *d_audio, const int64_t *offsets, int32_t count, int32_t frames,
                                         float *d_waveform, float *d_mask);

/* A set of sessions for a segmentation model of `frames` frames per chunk (1 .. 2^20). */
fa_status fa_od_create(int32_t frames, fa_od_databases **out);
void fa_od_destroy(fa_od_databases *h);
/* A new session: an empty database whose next new id is 1. */
fa_status fa_od_open(fa_od_databases *h, int32_t *session);
fa_status fa_od_close(fa_od_databases *h, int32_t session);

/* After the segmentation model: logits [count x F x 7] for sessions[0 .. count).  Writes each local speaker's
 * clean-frame mask repeat-padded from numMasksInChunk = min((F * chunk_size + 80000) / 160000, F) entries
 * (masks, [count x 3 x F]) and need[count x 3]: 1 where the embedding model runs (the mask sums to at least
 * min_active_frames_count), 0 where its embedding is zero.  The decoded frames stay staged for fa_od_advance.
 * The powerset argmax takes the first index of the maximum; a NaN logit is never chosen past index 0.  One launch. */
fa_status fa_od_embedding_inputs(fa_od_databases *h, int32_t count, const int32_t *sessions, const float *logits,
                                 const fa_od_config *cfg, float *masks, int32_t *need);
fa_status fa_od_embedding_inputs_device(fa_od_databases *h, int32_t count, const int32_t *sessions,
                                        const float *d_logits, const fa_od_config *cfg, float *d_masks,
                                        int32_t *d_need);
/* After the embedding model: embeddings [count x 3 x 256] (the rows of local speakers whose need was 0 are never read) and each chunk's offset in
 * seconds.  Assigns local speakers 0, 1, 2 in order, then writes assigned[count x 3 x 2] = (named, key) of each local
 * speaker's id, or (-1, 0) for none; seg_counts[count]; and per session up to 3 * ((F + 1) / 2) segments:
 * seg_ids [count x that x 2] (named, key) and seg_values [count x that x 3] (start, end, quality), in start order.
 * Every session named must have staged a chunk.  One launch and one synchronisation. */
fa_status fa_od_advance(fa_od_databases *h, int32_t count, const int32_t *sessions, const float *embeddings,
                        const double *chunk_offsets, const fa_od_config *cfg, int64_t *assigned, int32_t *seg_counts,
                        int64_t *seg_ids, float *seg_values);
fa_status fa_od_advance_device(fa_od_databases *h, int32_t count, const int32_t *sessions, const float *d_embeddings,
                               const double *chunk_offsets, const fa_od_config *cfg, int64_t *d_assigned,
                               int32_t *d_seg_counts, int64_t *d_seg_ids, float *d_seg_values);

/* Cosine distances [count x speakers] from `count` embeddings to every speaker of a session, in database order
 * (findSpeaker and findMatchingSpeakers rank these).  One launch. */
fa_status fa_od_query(fa_od_databases *h, int32_t session, int32_t count, const float *embeddings, float *distances);
fa_status fa_od_query_device(fa_od_databases *h, int32_t session, int32_t count, const float *d_embeddings,
                             float *d_distances);
/* The session's speaker count and next new id. */
fa_status fa_od_speaker_count(fa_od_databases *h, int32_t session, int64_t *count, int64_t *next_id);
/* Readback in database (insertion) order: speakers[count], current [count x 256], raws [count x 50 x 256] (oldest
 * first, zero past raw_count).  Any output may be NULL. */
fa_status fa_od_read(fa_od_databases *h, int32_t session, fa_od_speaker *speakers, float *current, float *raws);

/* initializeKnownSpeakers(_:mode:preserveIfPermanent:).  Speaker i is Speaker.init of speakers[i] with
 * current[i] (normalised on the way in) and speakers[i].raw_count raw embeddings, each RawEmbedding.init of its row
 * of raws (rows of all speakers packed in order; at most 50 per speaker).  Refused without change when an identity
 * repeats. */
fa_status fa_od_initialize(fa_od_databases *h, int32_t session, int32_t count, const fa_od_speaker *speakers,
                           const float *current, const float *raws, int32_t mode, int32_t preserve_if_permanent);
/* upsertSpeaker(_:): an existing id (named, key) takes duration, update_count, current (as given, not normalised) and
 * raw_count raws (each RawEmbedding.init of its row), and becomes permanent if `permanent` is set; a new id is
 * Speaker.init of the same fields, appended, and moves the next new id past its numeric value. */
fa_status fa_od_upsert(fa_od_databases *h, int32_t session, const fa_od_speaker *speaker, const float *current,
                       const float *raws);
/* removeSpeaker(_:keepIfPermanent:); *removed tells whether it did. */
fa_status fa_od_remove(fa_od_databases *h, int32_t session, int32_t named, int64_t key, int32_t keep_if_permanent,
                       int32_t *removed);
/* mergeSpeaker(_:into:stopIfPermanent:); *merged tells whether it did. */
fa_status fa_od_merge(fa_od_databases *h, int32_t session, int32_t source_named, int64_t source_key,
                      int32_t destination_named, int64_t destination_key, int32_t stop_if_permanent, int32_t *merged);
/* makeSpeakerPermanent (permanent 1) and revokePermanence (0); *found tells whether the speaker exists. */
fa_status fa_od_set_permanent(fa_od_databases *h, int32_t session, int32_t named, int64_t key, int32_t permanent,
                              int32_t *found);
/* reset(keepIfPermanent:) */
fa_status fa_od_reset(fa_od_databases *h, int32_t session, int32_t keep_if_permanent);

#ifdef __cplusplus
}
#endif

#endif
