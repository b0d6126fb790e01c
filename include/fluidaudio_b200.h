/* fluidaudio_b200 — C ABI of the H100-native (sm_90a) implementation of FluidAudio's two CPU hot paths.
 *
 * Every entry point is what a Swift/cgo/ctypes FFI binding for that piece of the reference would bind:
 * plain pointers and sizes, caller-owned buffers, an int status, no exception ever crosses the boundary
 * (same conventions as the reference's only C boundary, Sources/FastClusterWrapper/include/FastClusterWrapper.h).
 * There is NO CPU fallback: without an sm_90a device every compute call returns FA_NO_DEVICE.
 *
 * Reference interfaces replaced (paths relative to the FluidAudio repository):
 *   fa_mel_*             Sources/FluidAudio/Shared/AudioMelSpectrogram.swift:18-121 (class + init),
 *                        :132 compute, :185 computeFlat, :299/:325 computeFlatTransposed, :486-493 getters
 *   fa_audio_resample / fa_audio_to_mel / fa_resample_output_count
 *                        Sources/FluidAudio/Shared/AudioConverter.swift:60-71 (resample), :299-370 (convertBuffer),
 *                        :388-442 (linearResample) — the converter stage on the GPU, fused ahead of the log-mel kernel
 *   fa_linear_resample   Sources/FluidAudio/Shared/AudioConverter.swift:388-442 (linearResample; the converter stage's linear kernel)
 *   fa_l2_normalize_rows Sources/FluidAudio/Diarizer/Offline/Clustering/AHCClustering.swift:70-105
 *   fastcluster_compute_centroid_linkage  (declared in FastClusterWrapper.h, same symbol as the reference)
 *   fa_ahc_cluster       AHCClustering.swift:20-67  (AHCClustering.cluster)
 *   fa_dendrogram_cut    AHCClustering.swift:112-121,124-210
 *   fa_vbx_refine        Sources/FluidAudio/Diarizer/Offline/Clustering/VBxClustering.swift:41-165 (refine)
 *   fa_compute_centroids Sources/FluidAudio/Diarizer/Offline/Core/OfflineDiarizerManager.swift:613-691
 *   fa_assign_embeddings OfflineDiarizerManager.swift:789-822
 *   fa_diarize_cluster   OfflineDiarizerManager.swift:270-384 (cluster(_:), clustering phase)
 *   fa_constrained_assign / fa_hungarian_solve / fa_build_chunk_assignments
 *                        ConstrainedClusterAssignment.swift:20-42, HungarianAssignment.swift:8-97, :885-911
 *   fa_kmeans_cluster / fa_speaker_constraints_resolve
 *                        KMeansClustering.swift:39-130,212-223, SpeakerCountConstraints.swift:27-85,
 *                        VBxClustering.swift:685-733 (refineWithConstraints)
 *   fa_build_segments    Diarizer/Offline/Utils/OfflineReconstruction.swift:24-253, 359-505
 *   fa_seg_* / fa_embedding_plan / fa_embed_windows / fa_weight_resample
 *                        Diarizer/Offline/Segmentation/OfflineSegmentationProcessor.swift:55-56,118-190,321-405,
 *                        Diarizer/Offline/Extraction/OfflineEmbeddingExtractor.swift:421-707, WeightInterpolation.swift
 *                        (the arithmetic of OfflineDiarizerManager.prepare around the two networks)
 *   fa_diarizer_timeline_*  Diarizer/DiarizerTimeline.swift:801-1336 (addChunk, finalize, reset, updateSegments)
 *   fa_export_*          OfflineDiarizerManager.swift:913-955 (exportEmbeddings: the JSON dump of TimedEmbedding +
 *                        cluster, OfflineDiarizerTypes.swift:706-716) — the backend's on-disk input format
 */
#ifndef FLUIDAUDIO_B200_H
#define FLUIDAUDIO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    FA_STATUS_OK = 0,
    FA_STATUS_INVALID_ARGUMENT = 1,
    FA_STATUS_INDEX_OVERFLOW = 2,
    FA_STATUS_OUTPUT_TOO_SMALL = 3,
    FA_STATUS_ALLOCATION_FAILURE = 4,
    FA_STATUS_RUNTIME_ERROR = 5,   /* e.g. NaN distance, as the reference's nan_error */
    FA_STATUS_NO_DEVICE = 6,       /* no sm_90a GPU visible: there is deliberately no CPU fallback */
    FA_STATUS_CUDA_ERROR = 7,
    FA_STATUS_UNSUPPORTED = 8,
    FA_STATUS_UNKNOWN_ERROR = 255
} fa_status;

/* ---- runtime ------------------------------------------------------------------------------------------- */
const char *fa_version(void);
/* Thread-local text of the last failure.  After any call that fails (a status other than FA_STATUS_OK, or -1 from a
 * counting call), the text describes that call's failure; a call that succeeds leaves the text unchanged. */
const char *fa_last_error(void);
int32_t fa_device_count(void);              /* sm_90a devices visible */
fa_status fa_set_device(int32_t ordinal);   /* binds the calling thread; one process per GPU is the intended use */
fa_status fa_device_synchronize(void);
int64_t fa_kernel_launch_count(void);       /* kernels this library has launched in this process */

/* Pinned host memory and device memory for callers that want the copy engines / resident buffers. */
fa_status fa_host_alloc(size_t bytes, void **out);
fa_status fa_host_free(void *p);
fa_status fa_device_alloc(size_t bytes, void **out);
fa_status fa_device_free(void *p);
fa_status fa_memcpy_h2d(void *dst_device, const void *src_host, size_t bytes);
fa_status fa_memcpy_d2h(void *dst_host, const void *src_device, size_t bytes);

/* Bare copy-engine probe: `reps` rounds of one H2D copy (h2d_bytes from host_src) and one D2H copy (d2h_bytes into
 * host_dst) issued together on two streams; *ms_per_round = wall clock per round.  The floor under every host-buffer
 * ("end to end") number: what PCIe and the host memory path deliver with no kernel in between. */
fa_status fa_memcpy_probe(const void *host_src, size_t h2d_bytes, void *host_dst, size_t d2h_bytes, int32_t reps,
                          float *ms_per_round);

/* Device-side timing of a region on the library's default stream (CUDA events). */
fa_status fa_timer_start(void);
fa_status fa_timer_stop_ms(float *elapsed_ms);

/* ---- log-mel frontend ---------------------------------------------------------------------------------- */
typedef struct {
    int32_t sample_rate;     /* 16000 */
    int32_t n_mels;          /* 128 (reference default); 80 in BASELINE config 2 */
    int32_t n_fft;           /* 512 */
    int32_t hop_length;      /* 160 */
    int32_t win_length;      /* 400 */
    float preemph;           /* 0.97 */
    int32_t pad_to;          /* 0 -> 1 */
    float log_floor;         /* 2^-24 */
    int32_t log_floor_mode;  /* 0 = additive log(x+floor), 1 = clamped log(max(x,floor)) */
    int32_t window_periodic; /* 0 = symmetric Hann, 1 = periodic */
} fa_mel_config;

enum { FA_MEL_PAD_CENTER = 0, FA_MEL_PAD_PREPADDED = 1, FA_MEL_LEGACY_COMPUTE = 2 };
enum { FA_MEL_TIME_MAJOR = 0 /* [T x nMels], computeFlatTransposed */, FA_MEL_MEL_MAJOR = 1 /* [nMels x T], computeFlat / compute */ };

typedef struct fa_mel fa_mel;   /* one handle per stream of calls: like the Swift class it is not thread-safe */

void fa_mel_default_config(fa_mel_config *cfg);
fa_status fa_mel_create(const fa_mel_config *cfg, fa_mel **out);

/* The other STFT -> mel -> log frontends of the reference, as a superset of fa_mel_config.  A handle made by
 * fa_mel_create_ex is an ordinary fa_mel: every fa_mel_compute* call, fa_audio_to_mel, the timers and the getters work
 * on it.  Reflect padding, spectrum_power != 2 and the affine epilogue run on the any-nFFT kernel; fa_mel_stream_*,
 * fa_mel_unified_features and fa_mel_lseend_features refuse a handle whose ex fields are not neutral
 * (FA_STATUS_INVALID_ARGUMENT).  A handle from fa_mel_ex_default_config equals fa_mel_create on the same base.
 *   FA_MEL_FB_AUDIO_MEL  AudioMelSpectrogram's Slaney table (Shared/AudioMelSpectrogram.swift:564-642)
 *   FA_MEL_FB_COHERE     CohereMelSpectrogram.slaneyMelFilter, f_min .. f_max (ASR/Cohere/CoherePipeline.swift:273-303);
 *                        also its window: symmetric Hann with a length-1 window [0] (:90-97)
 *   FA_MEL_FB_STYLETTS2  StyleTTS2MelExtractor.htkMelFilterbank, float32, bins k * filter_sample_rate / nFFT
 *                        (TTS/StyleTTS2/Pipeline/Preprocess/StyleTTS2MelExtractor.swift:174-221)
 *   FA_MEL_FB_LUXTTS     LuxTtsMelExtractor.htkMelFilterbank, float64 (TTS/LuxTts/LuxTtsMelExtractor.swift:160-187)
 * FA_MEL_EDGE_REFLECT changes what FA_MEL_PAD_CENTER pads with: audio index i < 0 reads x[min(-i, n-1)], i >= n reads
 * x[max(2n-2-i, 0)] (the reference's reflectPad clamps, :226-250), an empty clip reads zeros.  It needs preemph 0. */
enum { FA_MEL_FB_AUDIO_MEL = 0, FA_MEL_FB_COHERE = 1, FA_MEL_FB_STYLETTS2 = 2, FA_MEL_FB_LUXTTS = 3 };
enum { FA_MEL_EDGE_ZERO = 0, FA_MEL_EDGE_REFLECT = 1 };
typedef struct {
    fa_mel_config base;          /* sample_rate = the audio's rate (and the converter stage's target rate) */
    int32_t filterbank;          /* FA_MEL_FB_*: whose table construction, restated exactly */
    int32_t filter_sample_rate;  /* rate the bin frequencies are computed for; 0 = base.sample_rate (StyleTTS2: 16000) */
    float f_min, f_max;          /* Hz; f_max <= 0 means filter_sample_rate / 2 (Cohere only; the others fix 0 .. sr/2) */
    int32_t center_edge;         /* what .center pads with: zeros (default) or reflection */
    float spectrum_power;        /* 2 = |X|^2 (default), 1 = |X|, any other p > 0 = |X|^p */
    float log_mean, log_std;     /* out = (log(..) - log_mean) / log_std; 0 / 1 (default) skips it */
} fa_mel_ex_config;
void fa_mel_ex_default_config(fa_mel_ex_config *cfg);   /* base = fa_mel_default_config, everything else neutral */
void fa_mel_preset_cohere(fa_mel_ex_config *cfg);       /* CohereMelSpectrogram.Config() + CohereAsrConfig */
void fa_mel_preset_styletts2(fa_mel_ex_config *cfg);    /* StyleTTS2Constants */
void fa_mel_preset_luxtts(fa_mel_ex_config *cfg);       /* LuxTtsConstants */
/* Anything the kernels cannot honour is refused before any allocation, with fa_last_error text. */
fa_status fa_mel_create_ex(const fa_mel_ex_config *cfg, fa_mel **out);

/* The reference classes' own calls, one mel launch each (plus the CMVN epilogue for Cohere).  Each needs a handle of its
 * class (filterbank kind, edge, spectrum and log mode; pad_to 0 or 1), else FA_STATUS_INVALID_ARGUMENT; a too small
 * out_len gives FA_STATUS_OUTPUT_TOO_SMALL.  Both are returned before any copy or launch, with out untouched.
 * fa_mel_cohere_features = CohereMelSpectrogram.compute + padOrTruncate (CoherePipeline.swift:127-263): T = 1 + n / hop
 *   frames, valid = n / hop, per-mel CMVN (ddof 1, epsilon 1e-5) over all valid frames when valid > 1, frames >= valid
 *   zeroed, out = [n_mels x W] with W = fixed_frames (truncated or zero-padded), or W = T when fixed_frames < 0;
 *   *frames = W, *valid_frames = min(valid, W).  Pre-emphasis runs as one fused multiply-add per sample where the
 *   reference rounds twice (see DESIGN §4.1b).
 * fa_mel_styletts2_features = StyleTTS2MelExtractor.compute: [n_mels x frames], frames = 1 + n / hop (1 for n = 0).
 * fa_mel_luxtts_features = LuxTtsMelExtractor.extract: [frames x n_mels], frames = (n + hop/2) / hop (0 when n == 0). */
fa_status fa_mel_cohere_features(fa_mel *mel, const float *audio, size_t n, int64_t fixed_frames, float *out,
                                 size_t out_len, int64_t *frames, int64_t *valid_frames);
fa_status fa_mel_styletts2_features(fa_mel *mel, const float *audio, size_t n, float *out, size_t out_len,
                                    int64_t *frames);
fa_status fa_mel_luxtts_features(fa_mel *mel, const float *audio, size_t n, float *out, size_t out_len, int64_t *frames);
void fa_mel_destroy(fa_mel *mel);
fa_status fa_mel_get_window(const fa_mel *mel, float *out, size_t len);       /* getHannWindow(): win_length floats */
fa_status fa_mel_get_filterbank(const fa_mel *mel, float *out, size_t len);   /* getFilterbank(): n_mels x (n_fft/2+1) */
/* frames the reference would produce; expected_frames < 0 means nil */
int64_t fa_mel_frame_count(const fa_mel *mel, int64_t sample_count, int32_t padding_mode, int64_t expected_frames);

/* Arithmetic of the 512-point transform (window product, |.|^2, filterbank and log are float32 in both, like the reference):
 *   FA_MEL_PRECISION_F64  (default) DFT evaluated in FP64 and rounded once — the implementation-independent value,
 *                         reproduces the oracle to ~5e-6 in the log domain whatever the signal's dynamic range;
 *   FA_MEL_PRECISION_F32  DFT in float32 like the reference's own vDSP_DFT_zop (AudioMelSpectrogram.swift:459-481), two
 *                         frames per warp in float32 arithmetic instead of FP64; carries the float32 noise floor of
 *                         any float32 FFT (measured max |delta log-mel| 6e-5 over BASELINE's hour of audio). */
enum { FA_MEL_PRECISION_F64 = 0, FA_MEL_PRECISION_F32 = 1 };
fa_status fa_mel_set_precision(fa_mel *mel, int32_t precision);
int32_t fa_mel_get_precision(const fa_mel *mel);
/* Host-buffer calls on long clips are cut into `chunks` units whose H2D copy, kernels and D2H copy overlap on three
 * streams (default 24; 1 = no overlap).  Results do not depend on it. */
fa_status fa_mel_set_pipeline_chunks(fa_mel *mel, int32_t chunks);
/* When the caller's time-major output buffer is pinned host memory (fa_host_alloc / cudaHostAlloc), the kernel stores its rows
 * straight into it over PCIe instead of staging them in HBM and copying.  Default OFF: the copy engine is the
 * measured default; pageable buffers always take the copy.  Any 4-byte aligned `out` works (16-byte aligned rows are
 * stored as 16-byte vectors, other rows one float at a time); results are identical either way. */
fa_status fa_mel_set_zero_copy_output(fa_mel *mel, int32_t enabled);

/* Host buffers in and out (the drop-in call).  On return *mel_length = valid frames, *num_frames = padded frames;
 * out receives num_frames*n_mels floats in `layout`.  Mirrors computeFlatTransposed / computeFlat / compute. */
fa_status fa_mel_compute(fa_mel *mel, const float *audio, size_t sample_count, float last_audio_sample,
                         int32_t padding_mode, int64_t expected_frames, int32_t layout, float *out, size_t out_len,
                         int64_t *mel_length, int64_t *num_frames);
/* Same with buffers already resident in HBM (asynchronous on the library stream).  d_audio and d_out need only 4-byte
 * (float) alignment; 16-byte aligned buffers take the faster bulk-copy input and vector stores, with identical results.
 * As in every mel entry point: any hop is accepted (nFFT 512 with an even hop takes the specialised kernel while its shared
 * memory fits, everything else the any-nFFT kernel), and a NaN sample makes every frame whose window holds it (after
 * pre-emphasis) NaN in every mel with a non-empty filter band, in both log-floor modes. */
fa_status fa_mel_compute_device(fa_mel *mel, const float *d_audio, size_t sample_count, float last_audio_sample,
                                int32_t padding_mode, int64_t expected_frames, int32_t layout, float *d_out,
                                size_t out_len, int64_t *mel_length, int64_t *num_frames);
/* Batch of independent clips.  Clip i is audio[offsets[i] .. offsets[i+1]); its output starts at out_offsets[i]
 * and holds num_frames[i]*n_mels floats (use fa_mel_frame_count to size it).  last_samples may be NULL. */
fa_status fa_mel_compute_batch(fa_mel *mel, const float *audio, const int64_t *offsets, int32_t clip_count,
                               const float *last_samples, int32_t padding_mode, int32_t layout, float *out,
                               const int64_t *out_offsets, int64_t *mel_lengths, int64_t *num_frames);
/* The batch with buffers resident in HBM.  offsets and out_offsets may be any float offsets (d_audio and d_out 4-byte
 * aligned); results are identical to fa_mel_compute_batch. */
fa_status fa_mel_compute_batch_device(fa_mel *mel, const float *d_audio, const int64_t *offsets, int32_t clip_count,
                                      const float *last_samples, int32_t padding_mode, int32_t layout, float *d_out,
                                      const int64_t *out_offsets, int64_t *mel_lengths, int64_t *num_frames);

/* Live streams: SortformerDiarizer's incremental mel stream (Diarizer/Sortformer/SortformerDiarizer.swift:204-217
 * resetMelStreamLocked, :417-424 addAudio, :842-870 preprocessAudioToFeaturesLocked / emitMelFramesLocked, :876-901
 * padAndEmitRemainingMelLocked) for many sessions on one handle, which they share config, precision and streams with.
 * A session starts with nFFT/2 zero samples buffered.  A push appends its samples and emits every frame whose window they
 * cover: count = (received - win/2) / hop + 1 - emitted, the .prePadded log-mel of the buffer with expected_frames = count
 * and the session's last_audio_sample, after which count*hop samples are dropped.  finish (after the push's samples)
 * appends nFFT/2 samples of the decay value *= preemph (zeros for preemph 0) and emits the frames left up to the .center
 * count 1 + (received + nFFT - win) / hop; later pushes to a finished session are ignored.  Only configurations with
 * pad_to <= 1 and hop_length <= win_length open a session (else FA_STATUS_INVALID_ARGUMENT).
 *   fa_mel_stream_open     resets and returns the lowest free id (ids are dense from 0 and reused after close).
 *   fa_mel_stream_frames   rows the next push of new_samples (finish 0/1) to `session` emits; -1 for a bad handle / session.
 *   fa_mel_stream_push     session sessions[i] receives audio[offsets[i] .. offsets[i+1]) (packed as in
 *                          fa_mel_compute_batch; count + 1 offsets), finished after them when finish[i] != 0 (finish may
 *                          be NULL).  The sessions of one push are distinct.  frames[i] receives session i's rows; out
 *                          receives them time-major in call order (session i at row sum_{j<i} frames[j]), out_len floats
 *                          must hold all of them.  Every argument is checked before any state changes: a failed push
 *                          leaves every session as it was.  One push costs one copy of the samples, one of the
 *                          descriptors, two kernel launches, one copy of the rows and one synchronisation, whatever the
 *                          number of sessions.
 *   fa_mel_stream_push_device  the same with d_audio / d_out in HBM, asynchronous on the handle's compute stream
 *                          (frames[] is still returned on return).
 * Rows equal fa_mel_compute(buffer, last, FA_MEL_PAD_PREPADDED, count) of the reference's buffer bit for bit.  Sessions are
 * not thread-safe, like the handle. */
fa_status fa_mel_stream_open(fa_mel *mel, int32_t *session);
fa_status fa_mel_stream_close(fa_mel *mel, int32_t session);
int64_t fa_mel_stream_frames(const fa_mel *mel, int32_t session, int64_t new_samples, int32_t finish);
fa_status fa_mel_stream_push(fa_mel *mel, int32_t count, const int32_t *sessions, const float *audio,
                             const int64_t *offsets, const int32_t *finish, float *out, size_t out_len, int64_t *frames);
fa_status fa_mel_stream_push_device(fa_mel *mel, int32_t count, const int32_t *sessions, const float *d_audio,
                                    const int64_t *offsets, const int32_t *finish, float *d_out, size_t out_len,
                                    int64_t *frames);

/* CUDA-event timer on the stream the mel kernels run on: bracket any number of fa_mel_compute*_device calls. */
fa_status fa_mel_timer_start(fa_mel *mel);
fa_status fa_mel_timer_stop_ms(fa_mel *mel, float *elapsed_ms);

/* Callers directly behind AudioMelSpectrogram, with their post-processing as device epilogues of the mel kernel.
 * fa_mel_unified_features = UnifiedMelExtractor.features(window:validCount:) (ASR/Parakeet/Unified/
 *   UnifiedMelExtractor.swift:52-113): the handle must be configured like its AudioMelSpectrogram (:31-40);
 *   total_frames = window_samples / hop + 1, valid_frames = min(valid_count / hop, total_frames); out receives the
 *   per-feature-normalised log-mel packed [n_mels x total_frames] (the MLMultiArray [1, nMels, T]).
 * fa_mel_lseend_features = LSEENDPreprocessor.processAudioQueue (Diarizer/LS-EEND/LSEENDPreprocessor.swift:249-283):
 *   the handle configured as :70-81 (preemph 0, periodic Hann, clamped floor 1e-10); out receives [frames x n_mels]
 *   log10-scaled, cumulative-mean-normalised features; cmn_mean[n_mels] / cmn_count are the running state, updated.
 * Both return exactly their frames, so both need a handle with pad_to 0 or 1 (the reference's padTo: 0); any other
 * pad_to gives FA_STATUS_INVALID_ARGUMENT before any copy or launch, with cmn_mean / cmn_count untouched. */
fa_status fa_mel_unified_features(fa_mel *mel, const float *window, size_t window_samples, size_t valid_count,
                                  float *out, size_t out_len, int64_t *total_frames, int32_t *valid_frames);
fa_status fa_mel_lseend_features(fa_mel *mel, const float *chunk, size_t n, float *cmn_mean, int64_t *cmn_count,
                                 float *out, size_t out_len, int64_t *frames);


/* NeMo per-feature normalisation of a time-major [frames x n_mels] buffer, in place (host buffer).
 * UnifiedMelExtractor.normalizePerFeature, Sources/FluidAudio/ASR/Parakeet/Unified/UnifiedMelExtractor.swift:88-113 */
fa_status fa_mel_normalize_per_feature(float *x, int64_t frames, int32_t n_mels, int64_t valid_frames);

/* ---- AudioConverter stage on the GPU ---------------------------------------------------------------------
 * PCM in any of the layouts AVAudioPCMBuffer / a WAV file hands over -> mono float32 at out_rate.
 *   algorithm AUTO follows AudioConverter.convertBuffer (:299-305): more than two channels take linearResample
 *   (:388-442, reproduced BIT FOR BIT: mean mixdown, src = i * ratio in double, two-tap float32 lerp); one or two
 *   channels take the AVAudioConverter path, whose arithmetic is closed — replaced by a documented Kaiser-windowed-sinc
 *   polyphase filter (24 zero crossings, beta 12, pass band 0.94 of the lower Nyquist; fluidaudio_b200/csrc/
 *   resample_plan.h), "parity unpinned" against Apple's sample values.  in_rate == out_rate is the identity on the
 *   samples (:66-68), after mixdown / int16 widening (v / 32768) when the input is not already mono float32.
 *   Output length = Int(Double(frames) / (in_rate / out_rate)) (:417-418) for both algorithms: the reference's tests
 *   accept +-1 % (AudioConverterTests.swift:129-176). */
enum { FA_PCM_F32 = 0, FA_PCM_I16 = 1 };
enum { FA_RESAMPLE_AUTO = 0, FA_RESAMPLE_SINC = 1, FA_RESAMPLE_LINEAR = 2 };
typedef struct {
    double in_rate;        /* e.g. 48000 */
    double out_rate;       /* 16000 (AudioConverter's default target) */
    int32_t channels;      /* >= 1 */
    int32_t format;        /* FA_PCM_F32 / FA_PCM_I16 */
    int32_t interleaved;   /* 1: [frames x channels] (WAV); 0: planar [channels x frames] (floatChannelData) */
    int32_t algorithm;     /* FA_RESAMPLE_* */
} fa_audio_format;
int64_t fa_resample_output_count(const fa_audio_format *fmt, int64_t frames);
/* AudioConverter.resample / resampleBuffer: host PCM in, host float32 mono out (conversion runs on the GPU). */
fa_status fa_audio_resample(const void *pcm, int64_t frames, const fa_audio_format *fmt, float *out, int64_t out_cap,
                            int64_t *out_count);
/* AudioConverter.resample followed by AudioMelSpectrogram.computeFlatTransposed / computeFlat as ONE device pipeline:
 * only the raw PCM crosses PCIe on the way in (int16 halves the bytes of the float path), the converted samples never
 * leave HBM.  fmt->out_rate must equal the handle's sample_rate.  *resampled_count (may be NULL) = samples at out_rate. */
fa_status fa_audio_to_mel(fa_mel *mel, const void *pcm, int64_t frames, const fa_audio_format *fmt,
                          float last_audio_sample, int32_t padding_mode, int32_t layout, float *out, size_t out_len,
                          int64_t *mel_length, int64_t *num_frames, int64_t *resampled_count);

/* AudioConverter.linearResample: planar [channels x frames] -> mono at out_rate.  Returns the sample count
 * through *out_count; call with out == NULL to size the buffer. */
fa_status fa_linear_resample(const float *planar, int64_t frames, int32_t channels, double in_rate, double out_rate,
                             float *out, int64_t out_cap, int64_t *out_count);

/* ---- offline clustering backend ------------------------------------------------------------------------ */
fa_status fa_l2_normalize_rows(const double *x, size_t rows, size_t dim, double *out);

/* AHCClustering.cluster: rows are NOT yet normalised; labels are canonical (first appearance order). */
fa_status fa_ahc_cluster(const double *features, size_t count, size_t dim, double threshold, int32_t *labels);

/* Device time of the calling thread's most recent linkage: [0] initial nearest-neighbour pass, [1] heapify + copies,
 * [2] persistent merge kernel, [3] total (ms).  Diagnostics only. */
void fa_ahc_last_stage_ms(float *out4);

/* Swift-side dendrogram cut + relabel on a SciPy-format linkage Z [(count-1) x 4]. */
fa_status fa_dendrogram_cut(const double *Z, size_t count, double threshold, int32_t *labels);

typedef struct {
    double Fa;               /* 0.07 */
    double Fb;               /* 0.8 */
    int32_t max_iterations;  /* 20 */
    double epsilon;          /* 1e-4 */
    double init_smoothing;   /* 7.0 */
} fa_vbx_config;
void fa_vbx_default_config(fa_vbx_config *cfg);

/* VBxClustering.refine.  rho: T x D; psi: psi_len doubles (identity if psi_len != D); initial: T labels.
 * speakers = number of distinct initial labels (the caller sizes gamma [T x speakers], pi [speakers],
 * elbos [max(max_iterations,1)], hard [T]).  *iterations receives the number of EM iterations run. */
fa_status fa_vbx_refine(const double *rho, size_t T, size_t D, const double *psi, size_t psi_len,
                        const int32_t *initial, int32_t speakers, const fa_vbx_config *cfg, double *gamma,
                        double *pi, double *elbos, int32_t *hard, int32_t *iterations);

/* computeCentroids (gamma/pi weighted, speakers with pi > 1e-7).  centroids capacity speakers x dim.
 * *centroid_count receives K. */
fa_status fa_compute_centroids(const double *embeddings, size_t T, size_t dim, const double *gamma, const double *pi,
                               int32_t speakers, double *centroids, int32_t *centroid_count);

/* assignEmbeddings: cosine against every centroid, first maximum wins.  scores may be NULL (else N x K). */
fa_status fa_assign_embeddings(const double *embeddings, size_t N, size_t dim, const double *centroids, int32_t K,
                               int32_t *labels, double *scores);

#define FA_NO_VALUE INT32_MIN   /* an absent optional count (Swift nil) in fa_cluster_config / fa_speaker_constraints_resolve */

typedef struct {
    double threshold;        /* 0.6  OfflineDiarizerConfig.clusteringThreshold */
    fa_vbx_config vbx;       /* warmStartFa/Fb, VBx.maxIterations, convergenceTolerance */
    /* OfflineDiarizerConfig.Clustering.numSpeakers / minSpeakers / maxSpeakers (OfflineDiarizerTypes.swift);
     * FA_NO_VALUE = nil (zero and negative counts are legal inputs, the reference clamps them to 1).
     * When the count VBx arrives at violates them the embeddings are re-clustered with K-Means (n_init 10, seeds 0..9,
     * 100 iterations) and assigned by plain argmax (VBxClustering.swift:685-733, OfflineDiarizerManager.swift:354-375). */
    int32_t num_speakers, min_speakers, max_speakers;
    int32_t reserved;
} fa_cluster_config;
void fa_cluster_default_config(fa_cluster_config *cfg);

typedef struct {
    int32_t training_count;    /* embeddings that survived the NaN/Inf filter */
    int32_t initial_clusters;  /* AHC cluster count (= VBx speaker count S) */
    int32_t vbx_iterations;
    int32_t centroid_count;    /* K */
    float ms_normalize, ms_ahc, ms_cut, ms_vbx, ms_assign, ms_total;   /* device/host stage times */
    int32_t was_adjusted;      /* VBxOutput.wasAdjusted: K-Means replaced the VBx clusters */
    int32_t detected_clusters; /* VBxOutput.assignedClusterCount before the adjustment */
} fa_cluster_info;

/* OfflineDiarizerManager.cluster(_:) lines 286-375 (unconstrained argmax assignment):
 *   emb256: N x emb_dim float32; rho: N x rho_dim float64; psi: rho_dim doubles, or NULL for the identity (pass NULL
 *   when the PLDA parameters have another length: VBxClustering.swift:71-76).  labels: N final assignments.
 * Optional outputs (may be NULL): initial [N] AHC labels of the training rows (-1 for filtered rows),
 * centroids [max_centroids x emb_dim], info. */
fa_status fa_diarize_cluster(const float *emb256, const double *rho, size_t N, size_t emb_dim, size_t rho_dim,
                             const double *psi, const fa_cluster_config *cfg, int32_t *labels, int32_t *initial,
                             double *centroids, int32_t max_centroids, fa_cluster_info *info);

/* Same with the reference's DEFAULT assignment (OfflineDiarizerConfig.Clustering.constrainedAssignment = true,
 * OfflineDiarizerManager.swift:357-369): chunk_index[N] is TimedEmbedding.chunkIndex; local speakers that share a chunk
 * are matched to distinct clusters (labels[i] = -2 when a chunk has more local speakers than clusters).
 * chunk_index == NULL, or a single centroid, falls back to the plain argmax like the reference. */
fa_status fa_diarize_cluster_chunks(const float *emb256, const double *rho, size_t N, size_t emb_dim, size_t rho_dim,
                                    const double *psi, const fa_cluster_config *cfg, const int32_t *chunk_index,
                                    int32_t *labels, int32_t *initial, double *centroids, int32_t max_centroids,
                                    fa_cluster_info *info);

/* HungarianAssignment.solve / maxScoreAssignment (HungarianAssignment.swift:8-61, :67-97),
 * ConstrainedClusterAssignment.assign (ConstrainedClusterAssignment.swift:20-42) and
 * OfflineDiarizerManager.buildChunkAssignments (:885-911).  Exact integer logic on tiny per-chunk matrices: host. */
fa_status fa_hungarian_solve(const int64_t *cost_square, int32_t n, int32_t *assignment);
fa_status fa_max_score_assignment(const double *scores, int32_t rows, int32_t cols, int32_t *assignment);
fa_status fa_constrained_assign(const double *scores, size_t N, int32_t K, const int32_t *chunk_index, int32_t *labels);
fa_status fa_build_chunk_assignments(const int32_t *chunk_index, const int32_t *speaker_index, const int32_t *assignments,
                                     size_t N, int32_t num_chunks, int32_t num_speakers, int32_t cluster_count,
                                     int32_t *matrix);

/* OfflineReconstruction.buildSegments (Diarizer/Offline/Utils/OfflineReconstruction.swift:24-253): the step after
 * fa_build_chunk_assignments in OfflineDiarizerManager.cluster(_:).  speaker_weights: SegmentationOutput.speakerWeights
 * flattened [num_chunks x num_frames x num_speakers]; chunk_offsets: SegmentationOutput.chunkOffsets (offsets_count may
 * be smaller than num_chunks: missing chunks start at chunk * window_duration); hard_clusters: the matrix returned by
 * fa_build_chunk_assignments [hard_rows x num_speakers] (-2 = inactive); centroid_count: centroids.count.
 * Output: *segment_count segments sorted by start (speakerId = "S<cluster+1>", embedding = centroid[cluster]); when
 * segment_cap is too small the first segment_cap are written and FA_STATUS_OUTPUT_TOO_SMALL is returned.  Host code; the
 * zero-vote re-embed pass (off by default, needs the embedding model) is not part of it.  speaker_weights and
 * chunk_offsets are what fa_seg_decode and fa_seg_windows produce. */
typedef struct {
    double frame_duration, window_duration, min_gap_duration, seg_min_duration_off, seg_min_duration_on, min_segment_duration;
    int32_t exclusive_segments;
    int32_t reserved;
} fa_reconstruct_config;
void fa_reconstruct_default_config(fa_reconstruct_config *cfg);   /* OfflineDiarizerConfig defaults, frame_duration = 0 */
fa_status fa_build_segments(const float *speaker_weights, int32_t num_chunks, int32_t num_frames, int32_t num_speakers,
                            const double *chunk_offsets, int32_t offsets_count, const int32_t *hard_clusters,
                            int32_t hard_rows, int32_t centroid_count, const fa_reconstruct_config *cfg,
                            int32_t *seg_cluster, float *seg_start, float *seg_end, float *seg_quality,
                            int32_t segment_cap, int32_t *segment_count);

/* OfflineReconstruction.buildSpeakerDatabase (:296-357): database [K x dim] = per speaker the float32 mean of its segments'
 * embeddings (a segment's embedding is Float(centroids[cluster])); segment_counts [K]; speakers without segment stay zero. */
fa_status fa_build_speaker_database(const int32_t *seg_cluster, int32_t segment_count, const double *centroids, int32_t K,
                                    int32_t dim, float *database, int32_t *segment_counts);

/* ---- offline diarization, prepare stage -------------------------------------------------------------------
 * The arithmetic of OfflineDiarizerManager.prepare around the two networks (which run outside this library):
 *   audio -> fa_seg_windows -> segmentation network -> fa_seg_decode -> fa_embedding_plan (+ fa_embed_windows)
 *         -> embedding network, PLDA -> fa_diarize_cluster_chunks -> fa_build_chunk_assignments -> fa_build_segments.
 * Reference (under Sources/FluidAudio/Diarizer/Offline): Segmentation/OfflineSegmentationProcessor.swift:55-56,118-190,
 * 303,321-405; Extraction/OfflineEmbeddingExtractor.swift:338-351,381-387,421-707,807-842; Extraction/
 * WeightInterpolation.swift:19-146; Utils/VDSPOperations.swift:142-155.
 *
 * Each call runs on a context leased from the library's pool and has finished when it returns.  The `_device` twins
 * take device pointers for the large buffers (audio, windows, logits, log-probabilities, weights and every per-entry
 * output) and leave them on the device; work queued on other streams that produces their inputs must have finished before the
 * call.  Small arrays (chunk offsets, chunk indices, the histogram, counts) are host memory in both.
 * Weights, class histogram, entries, frames, times and both weight matrices equal the reference bit for bit for the
 * binary weights fa_seg_decode produces; log-probabilities depend on expf / logf (Apple's vvexpf is closed) and sums of
 * non-binary weights on a summation order (vDSP's is closed): both are "parity unpinned", see DESIGN §2. */
typedef struct {
    int32_t sample_rate;            /* 16000 */
    float speech_onset_threshold;   /* 0.5 */
    double window_duration;         /* 10.0 s */
    double step_ratio;              /* 0.2, in (0, 1] */
} fa_seg_config;
typedef struct {
    int32_t exclude_overlap;        /* 1: embeddingExcludeOverlap */
    float skip_threshold;           /* EmbeddingSkipStrategy.maskSimilarity(threshold); < 0 = .none (default) */
    double min_segment_duration;    /* 1.0 s */
    int32_t weight_frames;          /* weightFrameCount of the embedding network: 589 */
    int32_t audio_sample_count;     /* audioSampleCount of the fbank input: 160000 */
    int32_t fbank_batch;            /* min(modelBatchLimit, 32): 32 */
    int32_t reserved;
} fa_embed_plan_config;
void fa_seg_default_config(fa_seg_config *cfg);                 /* OfflineDiarizerConfig.Segmentation.community */
void fa_embed_plan_default_config(fa_embed_plan_config *cfg);   /* OfflineDiarizerConfig.Embedding.community */

/* samplesPerWindow, samplesPerStep and the number of windows stride(from: 0, to: total_samples, by: step) yields
 * (0 for no samples).  Outputs may be NULL.  Host arithmetic. */
fa_status fa_seg_window_count(int64_t total_samples, const fa_seg_config *cfg, int32_t *chunks, int64_t *window,
                              int64_t *step);
/* Windows first_chunk .. first_chunk + chunk_count - 1: out_windows [chunk_count x window], samples past the end of the
 * audio zero; chunk_offsets [chunk_count] (host, may be NULL) = offset / sample_rate.  total_samples == 0 is the
 * reference's noSpeechDetected: FA_STATUS_RUNTIME_ERROR.  One launch. */
fa_status fa_seg_windows(const float *audio, int64_t total_samples, const fa_seg_config *cfg, int32_t first_chunk,
                         int32_t chunk_count, float *out_windows, double *chunk_offsets);
fa_status fa_seg_windows_device(const float *d_audio, int64_t total_samples, const fa_seg_config *cfg,
                                int32_t first_chunk, int32_t chunk_count, float *d_out_windows, double *chunk_offsets);
/* logits [chunks x frames x classes], classes 1 .. 16 (classes past the 8 powerset classes decode as class 7, as the
 * reference does; a NaN logit never wins the argmax).  log_probs [chunks x frames x classes] (may be NULL);
 * speaker_weights [chunks x frames x 3]; class_histogram [8] and speech_frames (host, may be NULL).  One launch. */
fa_status fa_seg_decode(const float *logits, int32_t chunks, int32_t frames, int32_t classes, const fa_seg_config *cfg,
                        float *log_probs, float *speaker_weights, int64_t *class_histogram, int64_t *speech_frames);
fa_status fa_seg_decode_device(const float *d_logits, int32_t chunks, int32_t frames, int32_t classes,
                               const fa_seg_config *cfg, float *d_log_probs, float *d_speaker_weights,
                               int64_t *class_histogram, int64_t *speech_frames);
/* Which (chunk, local speaker) pairs get an embedding, and with which weights.  speaker_weights [chunks x frames x
 * speakers]; chunk_offsets (host) as in fa_build_segments: a missing or non-finite offset is chunk * window_duration;
 * frame_duration <= 0 means window_duration / max(1, frames).  Entries come chunk-major, speaker-minor; each per-entry
 * array has capacity chunks * speakers and may be NULL; rows of skipped pairs are not written.  reuse_of[i] is the entry
 * whose embedding entry i reuses under the skip strategy, else -1.  frame_weights [entries x frames] is
 * TimedEmbedding.frameWeights, model_weights [entries x weight_frames] the embedding network's weights input.
 * counters [4] (host, may be NULL): masks evaluated, empty, fallback, skipped.  Two launches, three with the skip
 * strategy.  frames * (speakers + 1) floats must fit a CTA's shared memory (FA_STATUS_UNSUPPORTED otherwise). */
fa_status fa_embedding_plan(const float *speaker_weights, int32_t chunks, int32_t frames, int32_t speakers,
                            const double *chunk_offsets, int32_t offsets_count, double frame_duration,
                            int64_t total_samples, const fa_seg_config *seg_cfg, const fa_embed_plan_config *plan_cfg,
                            int32_t *chunk_index, int32_t *speaker_index, int32_t *start_frame, int32_t *end_frame,
                            double *start_time, double *end_time, float *mask_sum, int32_t *used_fallback,
                            int32_t *reuse_of, float *frame_weights, float *model_weights, int32_t *entry_count,
                            int64_t *counters);
fa_status fa_embedding_plan_device(const float *d_speaker_weights, int32_t chunks, int32_t frames, int32_t speakers,
                                   const double *chunk_offsets, int32_t offsets_count, double frame_duration,
                                   int64_t total_samples, const fa_seg_config *seg_cfg,
                                   const fa_embed_plan_config *plan_cfg, int32_t *d_chunk_index, int32_t *d_speaker_index,
                                   int32_t *d_start_frame, int32_t *d_end_frame, double *d_start_time, double *d_end_time,
                                   float *d_mask_sum, int32_t *d_used_fallback, int32_t *d_reuse_of,
                                   float *d_frame_weights, float *d_model_weights, int32_t *entry_count,
                                   int64_t *counters);
/* The fbank input of chunks chunk_index[0 .. count) (host; NULL = chunks 0 .. count - 1): out [count x
 * audio_sample_count], row i = min(chunk length, audio_sample_count) samples from round(offset * sample_rate) clamped
 * to the audio, zeros after them (a chunk without audio gives a zero row).  One launch. */
fa_status fa_embed_windows(const float *audio, int64_t total_samples, const double *chunk_offsets, int32_t offsets_count,
                           const int32_t *chunk_index, int32_t count, const fa_seg_config *cfg,
                           int32_t audio_sample_count, float *out);
fa_status fa_embed_windows_device(const float *d_audio, int64_t total_samples, const double *chunk_offsets,
                                  int32_t offsets_count, const int32_t *chunk_index, int32_t count,
                                  const fa_seg_config *cfg, int32_t audio_sample_count, float *d_out);
/* WeightInterpolation.resample2D: rows [row_count x in_len] -> out [row_count x out_len] (host buffers), the input
 * itself when the lengths match.  Non-positive lengths give FA_STATUS_INVALID_ARGUMENT (the reference returns []). */
fa_status fa_weight_resample(const float *rows, int64_t row_count, int32_t in_len, int32_t out_len, float *out);

/* KMeansClustering.clusterWithCentroidsNInit (Diarizer/Offline/Clustering/KMeansClustering.swift:39-130) on raw
 * embeddings [N x D]: labels [N], centroids (normalised space) [min(num_clusters, N) x D] -> *centroid_rows rows;
 * *best_init = index of the winning seed.  n_init <= 1 runs the single seeded clustering (:39-92).
 * A NaN or Inf in a row makes the inertia of every run NaN: the base-seed run is then returned (*best_init = 0).
 * fa_speaker_constraints_resolve = SpeakerCountConstraints.resolve (SpeakerCountConstraints.swift:27-71);
 * FA_NO_VALUE = nil. */
fa_status fa_kmeans_cluster(const double *embeddings, size_t N, size_t D, int32_t num_clusters, int32_t max_iterations,
                            int32_t n_init, uint64_t base_seed, int32_t *labels, double *centroids,
                            int32_t centroid_cap, int32_t *centroid_rows, int32_t *best_init);
fa_status fa_speaker_constraints_resolve(int64_t num_embeddings, int64_t num_speakers, int64_t min_speakers,
                                         int64_t max_speakers, int64_t *resolved_min, int64_t *resolved_max);

/* Embedding-export files (JSON array written by the reference when OfflineDiarizerConfig.embeddingExportPath is set):
 * {chunkIndex, speakerIndex, startFrame, endFrame, startTime, endTime, embedding256[], rho128[], cluster} per entry.
 * fa_export_shape parses the file and reports the entry count and vector lengths; fa_export_read fills caller-owned
 * arrays (any output pointer may be NULL); fa_export_write produces a file the reference's Codable struct decodes.
 * float32 values round-trip bit-exactly (shortest-form decimal <-> strtof). */
fa_status fa_export_shape(const char *path, size_t *count, size_t *emb_dim, size_t *rho_dim);
fa_status fa_export_read(const char *path, size_t count, size_t emb_dim, size_t rho_dim, int32_t *chunk_index,
                         int32_t *speaker_index, int32_t *start_frame, int32_t *end_frame, double *start_time,
                         double *end_time, float *emb, double *rho, int32_t *cluster);
fa_status fa_export_write(const char *path, size_t count, size_t emb_dim, size_t rho_dim, const int32_t *chunk_index,
                          const int32_t *speaker_index, const int32_t *start_frame, const int32_t *end_frame,
                          const double *start_time, const double *end_time, const float *emb, const double *rho,
                          const int32_t *cluster);

/* Many independent embedding sets (meetings) on this GPU.  Set m is rows [set_offsets[m], set_offsets[m+1]).
 * Several sets are clustered concurrently on disjoint SM partitions.  set_offsets[0] must be >= 0 and the offsets
 * non-decreasing, else FA_STATUS_INVALID_ARGUMENT before any work.  An empty set (equal offsets) is skipped and its
 * infos[m] is zeroed; rows outside every set are not written. */
fa_status fa_diarize_cluster_batch(const float *emb256, const double *rho, const int64_t *set_offsets,
                                   int32_t set_count, size_t emb_dim, size_t rho_dim, const double *psi,
                                   const fa_cluster_config *cfg, int32_t *labels, fa_cluster_info *infos);

/* Same with the reference's default constrained assignment in every set (OfflineDiarizerManager.swift:357-369):
 * chunk_index[row] is TimedEmbedding.chunkIndex of that row, numbered inside its own set; NULL = plain argmax. */
fa_status fa_diarize_cluster_batch_chunks(const float *emb256, const double *rho, const int64_t *set_offsets,
                                          int32_t set_count, size_t emb_dim, size_t rho_dim, const double *psi,
                                          const fa_cluster_config *cfg, const int32_t *chunk_index, int32_t *labels,
                                          fa_cluster_info *infos);

/* ---- Sortformer streaming state: SortformerStateUpdater.swift (Diarizer/Sortformer), the state of
 * SortformerTypes.swift:270-327 and the padded model inputs of SortformerModelInference.swift:266-303, for many live
 * sessions in HBM.  numSpeakers = 4, preEncoderDims = 512 and maxIndex = 99999 are constants, as in the reference.
 *
 * fa_sortformer_config holds the `var` fields of SortformerConfig (SortformerTypes.swift:31-97).
 * fa_sortformer_default_config writes one of the reference's eight static configs (FA_SORTFORMER_*; an unknown preset
 * gives FA_STATUS_INVALID_ARGUMENT).  fa_sortformer_resolve_config applies the init's clamps (chunkLen >= 1,
 * spkcacheLen >= (1 + sil) * 4, update period in [chunkLen, fifoLen + chunkLen]) and create's checks: contexts, fifoLen
 * and sil >= 0, finite thresholds and rates, and (spkcacheLen + fifoLen + max_core + sil) * 4 < maxIndex.  max_core
 * (<= 0: chunkLen) is the largest coreFrames a push may carry; it sizes each session's FIFO (fifoLen + max_core rows) and
 * speaker cache before compression (spkcacheLen + fifoLen + max_core rows).  Neither needs a device.
 *
 * fa_sortformer_step plans one streamingUpdate from lengths alone, as every push does per session before anything runs:
 * lengths_in = {spkcacheLength, fifoLength, spkcachePreds exists}; out = {coreFrames, popOutLength (0: no overflow),
 * compression, spkcacheLength, fifoLength, spkcachePreds exists} after it.  FA_STATUS_INVALID_ARGUMENT when the reference
 * throws insufficientPredsLength / insufficientChunkLength (pred_rows < spkcache + fifo + lc + core + rc), a context is
 * negative, or coreFrames = emb_length - lc - rc is outside [0, max_core].
 *
 * Sessions (like fa_mel_stream_*): fa_sortformer_open returns the lowest free id with a fresh state (empty cache and
 * FIFO, no predictions, silence mean 0, count 0); close frees it.  Sessions and the handle are not thread-safe.
 *
 * fa_sortformer_update: session sessions[i] takes batch row i of the model's outputs, chunk_embs [count x emb_rows x
 * 512] with emb_lengths[i] valid rows (chunk_pre_encoder_lengths, host memory), preds [count x pred_rows x 4]
 * (probabilities) and left_context[i] / right_context[i].  NULL left_context is the streaming rule (chunk index > 0 ?
 * chunkLeftContext : 0, SortformerDiarizer.swift:553); NULL right_context is chunkRightContext.  Each session runs
 * streamingUpdate exactly: fifoPreds refresh, FIFO append, pop into the silence profile and the cache, compressSpkcache.
 * Its confirmed rows [coreFrames x 4] and tentative rows [rc x 4] are packed in call order into confirmed / tentative
 * (*_len floats); confirmed_rows[i] / tentative_rows[i] receive the counts.  Duplicate or closed sessions, the step's
 * errors above and outputs too small give FA_STATUS_INVALID_ARGUMENT before any state changes.  One push is one
 * descriptor upload and ONE kernel launch whatever the count (host variant: plus its copies and one synchronisation).
 * fa_sortformer_update_device takes d_chunk_embs / d_preds / d_confirmed / d_tentative in HBM and is asynchronous on the
 * handle's stream (the row counts are returned on return).
 *
 * fa_sortformer_model_inputs: the next model call's inputs for count sessions: spkcache [count x spkcacheLen x 512] and
 * fifo [count x fifoLen x 512], rows [0, length) of the state then zeros; the lengths go to spkcache_lengths /
 * fifo_lengths (host, may be NULL).  ONE kernel launch; _device writes d_spkcache / d_fifo asynchronously.
 *
 * fa_sortformer_session_state reads one session back (tests, checkpoints, inspection): spkcache [spkcacheLength x 512],
 * spkcache_preds [spkcacheLength x 4] (written only when info->has_spkcache_preds), fifo [fifoLength x 512], fifo_preds
 * [fifoLength x 4], mean_silence [512]; any pointer may be NULL.  Synchronous. */
enum {
    FA_SORTFORMER_DEFAULT = 0,
    FA_SORTFORMER_FAST_V2 = 1,
    FA_SORTFORMER_FAST_V2_1 = 2,
    FA_SORTFORMER_BALANCED_V2 = 3,
    FA_SORTFORMER_BALANCED_V2_1 = 4,
    FA_SORTFORMER_HIGH_CONTEXT_V2 = 5,
    FA_SORTFORMER_HIGH_CONTEXT_V2_1 = 6,
    FA_SORTFORMER_EFFICIENT_V2_1 = 7,
};
typedef struct {
    int32_t chunk_len, chunk_left_context, chunk_right_context, fifo_len, spkcache_len, spkcache_update_period,
        spkcache_sil_frames_per_spk;
    float silence_threshold, pred_score_threshold, scores_boost_latest, strong_boost_rate, weak_boost_rate,
        min_pos_scores_rate;
} fa_sortformer_config;
typedef struct {
    int32_t spkcache_length, fifo_length, has_spkcache_preds, has_fifo_preds;
    int64_t chunks, silence_frames;
} fa_sortformer_session_info;
typedef struct fa_sortformer fa_sortformer;

fa_status fa_sortformer_default_config(fa_sortformer_config *cfg, int32_t preset);
fa_status fa_sortformer_resolve_config(const fa_sortformer_config *cfg, int32_t max_core_frames,
                                       fa_sortformer_config *resolved, int32_t *resolved_max_core);
fa_status fa_sortformer_step(const fa_sortformer_config *cfg, int32_t max_core_frames, const int32_t *lengths_in,
                             int32_t emb_length, int32_t pred_rows, int32_t left_context, int32_t right_context,
                             int32_t *out);
fa_status fa_sortformer_create(const fa_sortformer_config *cfg, int32_t max_core_frames, fa_sortformer **out);
void fa_sortformer_destroy(fa_sortformer *h);
fa_status fa_sortformer_open(fa_sortformer *h, int32_t *session);
fa_status fa_sortformer_close(fa_sortformer *h, int32_t session);
fa_status fa_sortformer_update(fa_sortformer *h, int32_t count, const int32_t *sessions, const float *chunk_embs,
                               int32_t emb_rows, const float *preds, int32_t pred_rows, const int32_t *emb_lengths,
                               const int32_t *left_context, const int32_t *right_context, float *confirmed,
                               size_t confirmed_len, float *tentative, size_t tentative_len, int64_t *confirmed_rows,
                               int64_t *tentative_rows);
fa_status fa_sortformer_update_device(fa_sortformer *h, int32_t count, const int32_t *sessions,
                                      const float *d_chunk_embs, int32_t emb_rows, const float *d_preds,
                                      int32_t pred_rows, const int32_t *emb_lengths, const int32_t *left_context,
                                      const int32_t *right_context, float *d_confirmed, size_t confirmed_len,
                                      float *d_tentative, size_t tentative_len, int64_t *confirmed_rows,
                                      int64_t *tentative_rows);
fa_status fa_sortformer_model_inputs(fa_sortformer *h, int32_t count, const int32_t *sessions, float *spkcache,
                                     float *fifo, int32_t *spkcache_lengths, int32_t *fifo_lengths);
fa_status fa_sortformer_model_inputs_device(fa_sortformer *h, int32_t count, const int32_t *sessions, float *d_spkcache,
                                            float *d_fifo, int32_t *spkcache_lengths, int32_t *fifo_lengths);
fa_status fa_sortformer_session_state(fa_sortformer *h, int32_t session, fa_sortformer_session_info *info,
                                      float *spkcache, float *spkcache_preds, float *fifo, float *fifo_preds,
                                      float *mean_silence);

/* ---- Diarizer timelines: the numeric core of DiarizerTimeline (Sources/FluidAudio/Diarizer/DiarizerTimeline.swift),
 * which turns frame-wise speaker probabilities (Sortformer, LS-EEND, ...) into speech segments, for many live sessions
 * in HBM.  Speaker identity (names, ids, enrollment) and the per-speaker segment lists stay with the caller, as in the
 * reference's DiarizerSpeaker.  Unrelated to fa_build_segments, the offline diarizer's reconstruction.
 *
 * fa_diarizer_timeline_config holds DiarizerTimelineConfig's numeric fields (:9-164) with maxStoredFrames required
 * (the reference's nil, unlimited, is not offered).  fa_diarizer_timeline_default_config writes a preset:
 * FA_TIMELINE_PRESET_DEFAULT is default(numSpeakers:frameDurationSeconds:) with the given values, thresholds 0.5, no
 * padding or minimum durations, sigmoids; FA_TIMELINE_PRESET_SORTFORMER is sortformerDefault (4 speakers, 0.08 s).
 * Both store FA_TIMELINE_DEFAULT_STORED_FRAMES rows.  fa_diarizer_timeline_config_from_seconds sets the four frame
 * counts from seconds as the seconds initialiser (:139-163) does: Int(round(seconds / frameDurationSeconds)) in float32,
 * rounding half away from zero; FA_STATUS_INVALID_ARGUMENT when a result is not finite or outside int32 (Swift traps).
 * Neither needs a device.
 *
 * fa_diarizer_timeline_create checks the config (numSpeakers in 1..32; pads and minimum durations >= 0; finite
 * thresholds and frame duration; a known activity type; maxStoredFrames >= 0) and max_tentative_rows >= 0, the most
 * tentative rows one push may carry per session.  Sessions (like fa_sortformer_*): fa_diarizer_timeline_open returns
 * the lowest free id with a fresh timeline; close frees it.  Sessions and the handle are not thread-safe.
 *
 * fa_diarizer_timeline_push: session sessions[i] takes finalized_rows[i] rows of `finalized` and tentative_rows[i] rows
 * of `tentative` ([rows x numSpeakers] each, packed in call order: the layout fa_sortformer_update[_device] writes, so
 * its buffers and row counts pass straight through).  Each session runs addChunk (:827-872) exactly: the finalized rows
 * join the stored predictions (trimmed to maxStoredFrames, skipped when it is 0), the tentative rows replace the
 * session's, then updateSegments runs over the finalized rows from the finalized cursor, keeping its scratch, and over
 * the tentative rows on a copy of it with the trailing tentative segment.  The new segments go to finalized_segments and
 * tentative_segments; in each list a session's segments are speaker-major, then in frame order within a speaker, and
 * sessions follow in call order; finalized_counts[i] / tentative_counts[i] receive each session's counts.  The outputs
 * must hold the bound fa_diarizer_timeline_segment_bound gives for the row counts (*_capacity in segments).  Duplicate
 * or closed sessions, more than max_tentative_rows tentative rows (or more than 2^30 finalized rows) in a session, and
 * outputs below the bound give FA_STATUS_INVALID_ARGUMENT before any state changes.  One push is one descriptor upload
 * and TWO kernel launches whatever the count; the host variant returns after at most two synchronisations, one for the
 * counts and one for exactly the segments.
 * fa_diarizer_timeline_push_device takes every row, segment and count buffer in HBM and is asynchronous on the
 * handle's stream.  The input rows must be complete when it is called: rows another handle wrote (for instance
 * fa_sortformer_update_device) are ready after fa_device_synchronize; the library does not order streams across handles.
 *
 * fa_diarizer_timeline_segment_bound: the segments a push of these row counts may emit, per list: a session of n
 * finalized and m tentative rows contributes numSpeakers * (n > 0 ? n / 2 + 1 : 0) finalized and
 * numSpeakers * ((m + 1) / 2 + 1) tentative segments.  No device.
 *
 * fa_diarizer_timeline_finalize (:877-891): each session's tentative rows join the stored ones and the finalized cursor
 * passes them.  At most one kernel launch, none when no named session holds tentative rows.  The per-speaker move of
 * tentative segments to finalized ones is the caller's.  fa_diarizer_timeline_reset (:921-934): no predictions,
 * cursor 0, fresh scratches.  fa_diarizer_timeline_clear_speaker: a fresh scratch for one speaker slot, as
 * removeSpeaker(clearCurrentSegment: true) and upsertSpeaker(transferCurrentSegment: false) do (:1108-1111,
 * :1134-1136).  rebuild (:945-1003) is reset, push and, when isComplete, finalize.
 *
 * fa_diarizer_timeline_session_state reads one session back (tests, the caller's probability queries): info, the stored
 * rows [stored_frames x numSpeakers] (frames finalized_frames - stored_frames .. finalized_frames - 1), the tentative
 * rows [tentative_frames x numSpeakers] and the numSpeakers scratches; any pointer but info may be NULL.  Synchronous. */
enum { FA_TIMELINE_SIGMOIDS = 0, FA_TIMELINE_LOGITS = 1 };
enum { FA_TIMELINE_PRESET_DEFAULT = 0, FA_TIMELINE_PRESET_SORTFORMER = 1 };
#define FA_TIMELINE_DEFAULT_STORED_FRAMES 7500
typedef struct {
    int32_t num_speakers;
    float frame_duration_seconds, onset_threshold, offset_threshold;
    int32_t onset_pad_frames, offset_pad_frames, min_frames_on, min_frames_off;
    int32_t activity_type;       /* FA_TIMELINE_SIGMOIDS or FA_TIMELINE_LOGITS */
    int32_t max_stored_frames;
} fa_diarizer_timeline_config;
typedef struct {
    int64_t start_frame, end_frame;
    float activity;
    int32_t speaker;
} fa_diarizer_timeline_segment;
/* SegmentScratch (:649-661); a `.min` frame reads INT64_MIN */
typedef struct {
    int64_t start_frame, end_frame, unmerged_start_frame, active_frame_count, unmerged_active_frame_count;
    float activity_sum, unmerged_activity_sum;
    int32_t speaking, has_segment;
} fa_diarizer_timeline_scratch;
typedef struct {
    int64_t finalized_frames, stored_frames, tentative_frames;
} fa_diarizer_timeline_session_info;
typedef struct fa_diarizer_timeline fa_diarizer_timeline;

fa_status fa_diarizer_timeline_default_config(fa_diarizer_timeline_config *cfg, int32_t preset, int32_t num_speakers,
                                              float frame_duration_seconds);
fa_status fa_diarizer_timeline_config_from_seconds(fa_diarizer_timeline_config *cfg, float onset_pad_seconds,
                                                   float offset_pad_seconds, float min_duration_on,
                                                   float min_duration_off);
fa_status fa_diarizer_timeline_segment_bound(int32_t num_speakers, int32_t count, const int64_t *finalized_rows,
                                             const int64_t *tentative_rows, int64_t *finalized_bound,
                                             int64_t *tentative_bound);
fa_status fa_diarizer_timeline_create(const fa_diarizer_timeline_config *cfg, int32_t max_tentative_rows,
                                      fa_diarizer_timeline **out);
void fa_diarizer_timeline_destroy(fa_diarizer_timeline *h);
fa_status fa_diarizer_timeline_open(fa_diarizer_timeline *h, int32_t *session);
fa_status fa_diarizer_timeline_close(fa_diarizer_timeline *h, int32_t session);
fa_status fa_diarizer_timeline_push(fa_diarizer_timeline *h, int32_t count, const int32_t *sessions,
                                    const float *finalized, const int64_t *finalized_rows, const float *tentative,
                                    const int64_t *tentative_rows, fa_diarizer_timeline_segment *finalized_segments,
                                    size_t finalized_capacity, fa_diarizer_timeline_segment *tentative_segments,
                                    size_t tentative_capacity, int64_t *finalized_counts, int64_t *tentative_counts);
fa_status fa_diarizer_timeline_push_device(fa_diarizer_timeline *h, int32_t count, const int32_t *sessions,
                                           const float *d_finalized, const int64_t *finalized_rows,
                                           const float *d_tentative, const int64_t *tentative_rows,
                                           fa_diarizer_timeline_segment *d_finalized_segments, size_t finalized_capacity,
                                           fa_diarizer_timeline_segment *d_tentative_segments, size_t tentative_capacity,
                                           int64_t *d_finalized_counts, int64_t *d_tentative_counts);
fa_status fa_diarizer_timeline_finalize(fa_diarizer_timeline *h, int32_t count, const int32_t *sessions);
fa_status fa_diarizer_timeline_reset(fa_diarizer_timeline *h, int32_t count, const int32_t *sessions);
fa_status fa_diarizer_timeline_clear_speaker(fa_diarizer_timeline *h, int32_t session, int32_t speaker);
fa_status fa_diarizer_timeline_session_state(fa_diarizer_timeline *h, int32_t session,
                                             fa_diarizer_timeline_session_info *info, float *stored, float *tentative,
                                             fa_diarizer_timeline_scratch *scratch);

#ifdef __cplusplus
}
#endif
#endif /* FLUIDAUDIO_B200_H */
