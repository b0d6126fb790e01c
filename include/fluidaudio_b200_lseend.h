/* C ABI of the LS-EEND feature streams in libfluidaudio_b200.so, beside the main header it builds on (status codes,
 * FA_MEL_PRECISION_*).  Plain C11, like the other headers under include/. */
#ifndef FLUIDAUDIO_B200_LSEEND_H
#define FLUIDAUDIO_B200_LSEEND_H

#include "fluidaudio_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* LS-EEND feature streams: LSEENDFeatureProvider (Sources/FluidAudio/Diarizer/LS-EEND/LSEENDPreprocessor.swift:46-384),
 * the log-mel front of the LS-EEND model, for many live sessions in HBM.  It sits between the audio (at the model's rate:
 * compose with fa_audio_resample for any other) and the model, whose predictions fa_diarizer_timeline_* takes.  The
 * model and its recurrent state stay with the caller.
 *
 * fa_lseend_stream_config holds the LSEENDMetadata fields the provider reads (LSEENDTypes.swift:10-58) and the
 * transform precision (FA_MEL_PRECISION_*).  fa_lseend_stream_resolve checks it (sizes positive, context_size and
 * conv_delay >= 0, hop_length <= win_length, derived sizes below 2^28) and returns what the provider's init derives
 * (:46-114): n_fft = the next power of two >= win_length, mel_frames = (chunk_size - 1) * subsampling +
 * 2 * context_size + 1 rows per model-input chunk, chunk_mels = subsampling * chunk_size, mel_context = mel_frames -
 * chunk_mels (negative when the mel queue's right context is), chunk_samples = hop * chunk_mels, the audio queue's
 * left context n_fft / 2 and whole context n_fft - hop, flush_samples = (context_size + conv_delay * subsampling) * hop
 * + n_fft / 2, mask_length = conv_delay + chunk_size, and audio_capacity = chunk_samples + n_fft - hop, which a
 * session's unread audio stays below.  No device.  fa_lseend_stream_create also builds the provider's
 * AudioMelSpectrogram (:70-81: preemph 0, padTo 0, log floor 1e-10 clamped, periodic Hann), so it refuses what the mel
 * kernels cannot run (n_fft below 32, more than 512 mels: FA_STATUS_UNSUPPORTED).
 *
 * Sessions (like fa_sortformer_*): fa_lseend_stream_open returns the lowest free id with a fresh provider (n_fft / 2
 * zero samples queued, context_size zero mel rows, a zero running mean, decoderMaskEnd 0, no snapshot); close frees it.
 *
 * fa_lseend_stream_push: session sessions[i] receives audio[offsets[i] .. offsets[i+1]) (count + 1 offsets, as in
 * fa_mel_stream_push), then, when drain[i] != 0 (drain may be NULL), drainRightContextWithSilence (:158-180):
 * flush_samples zeros and the zeros up to the next audio-chunk boundary.  Then processAudioQueue (:249-279) runs: every
 * whole audio chunk is popped with its context, its .prePadded log-mel is scaled by 1 / ln 10 and normalised by the
 * running mean, and the rows join the mel queue.  Then every ready chunk is emitted (emitNextChunk, :185-202): mel_frames
 * rows, the next decoder-mask window (decoderMaskEnd advances by chunk_size, capped at mask_length) and its warm-up count
 * min(mask_length - decoderMaskEnd, chunk_size).  A drained session takes more audio afterwards like any other.
 * Outputs in call order (session i's chunks after those of sessions 0 .. i-1): features [chunks x mel_frames x n_mels],
 * masks [chunks x chunk_size] (0 or 1), warm-up counts [chunks]; *_len in elements.  chunks[i] receives session i's count;
 * fa_lseend_stream_chunks gives it in advance (-1 for a bad handle or session; no device).  Duplicate or closed sessions,
 * decreasing offsets, more than 2^40 samples for one session and outputs too small for the chunks give
 * FA_STATUS_INVALID_ARGUMENT before any state changes: a failed push leaves every session as it was.  One push is one
 * copy of the samples, one of the descriptors, FOUR kernel launches (ingest, log-mel, running mean, gather) and one copy
 * of each output whatever the number of sessions; ONE launch (ingest) when no session completes an audio chunk, none
 * when no session receives samples or a drain.  The host variant returns after one synchronisation.
 * fa_lseend_stream_push_device takes d_audio and the three outputs in HBM and is asynchronous on the handle's stream
 * (chunks[] is host memory, returned on return).  Features equal those of fa_mel_lseend_features over the reference's
 * popAllChunks slices, sliced by its mel queue, bit for bit.
 *
 * fa_lseend_stream_snapshot / rollback / reset act on a list of distinct open sessions with one kernel launch each.
 * snapshot (takeSnapshot, :206-218) keeps a copy of both queues, the running mean, cmnCount and decoderMaskEnd in the
 * session's slot, replacing any earlier one; rollback (:224-233) restores it (FA_STATUS_INVALID_ARGUMENT, nothing
 * changed, when a session has none) and keeps it for another rollback; reset (:236-245) makes the session fresh, its
 * snapshot kept.  fa_lseend_stream_session_state reads one session back, synchronously: info, its unread audio
 * [audio_samples], its unread mel rows [mel_rows x n_mels] and cmn_mean [n_mels]; any pointer but info may be NULL.
 * Sessions and the handle are not thread-safe. */
typedef struct {
    int32_t sample_rate, n_mels, hop_length, win_length;
    int32_t context_size, subsampling, chunk_size, conv_delay;
    int32_t precision;   /* FA_MEL_PRECISION_F64 or FA_MEL_PRECISION_F32 */
} fa_lseend_stream_config;
typedef struct {
    int32_t n_fft, mel_frames, chunk_mels, mel_context, chunk_samples, audio_left_context, audio_context, flush_samples,
        mask_length, audio_capacity;
} fa_lseend_stream_sizes;
typedef struct {
    int64_t audio_samples, mel_rows, cmn_count;
    int32_t decoder_mask_end, has_snapshot;
} fa_lseend_stream_session_info;
typedef struct fa_lseend_stream fa_lseend_stream;

fa_status fa_lseend_stream_resolve(const fa_lseend_stream_config *cfg, fa_lseend_stream_sizes *sizes);
fa_status fa_lseend_stream_create(const fa_lseend_stream_config *cfg, fa_lseend_stream **out);
void fa_lseend_stream_destroy(fa_lseend_stream *h);
fa_status fa_lseend_stream_open(fa_lseend_stream *h, int32_t *session);
fa_status fa_lseend_stream_close(fa_lseend_stream *h, int32_t session);
int64_t fa_lseend_stream_chunks(const fa_lseend_stream *h, int32_t session, int64_t new_samples, int32_t drain);
fa_status fa_lseend_stream_push(fa_lseend_stream *h, int32_t count, const int32_t *sessions, const float *audio,
                                const int64_t *offsets, const int32_t *drain, float *features, size_t features_len,
                                float *masks, size_t masks_len, int32_t *warmup, size_t warmup_len, int64_t *chunks);
fa_status fa_lseend_stream_push_device(fa_lseend_stream *h, int32_t count, const int32_t *sessions,
                                       const float *d_audio, const int64_t *offsets, const int32_t *drain,
                                       float *d_features, size_t features_len, float *d_masks, size_t masks_len,
                                       int32_t *d_warmup, size_t warmup_len, int64_t *chunks);
fa_status fa_lseend_stream_snapshot(fa_lseend_stream *h, int32_t count, const int32_t *sessions);
fa_status fa_lseend_stream_rollback(fa_lseend_stream *h, int32_t count, const int32_t *sessions);
fa_status fa_lseend_stream_reset(fa_lseend_stream *h, int32_t count, const int32_t *sessions);
fa_status fa_lseend_stream_session_state(fa_lseend_stream *h, int32_t session, fa_lseend_stream_session_info *info,
                                         float *audio, float *mel, float *cmn_mean);

#ifdef __cplusplus
}
#endif
#endif /* FLUIDAUDIO_B200_LSEEND_H */
