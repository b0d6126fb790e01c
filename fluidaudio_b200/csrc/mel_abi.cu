// C ABI of the log-mel plan (declared in include/fluidaudio_b200.h): the plan and its presets (mel_kernels.cu), the
// host-buffer pipelines (mel_pipeline.cu), live streams (mel_stream.cu) and the adapters (mel_adapters.cu).  Every
// entry point that returns a status returns through guard() (c_abi.h).
#include "c_abi.h"
#include "call_context.h"
#include "mel_plan.h"

#include <cmath>
#include <cstring>
#include <memory>

struct fa_mel {
    fa::mel::MelPlan plan;
    fa::mel::MelStreamSet sessions;   // fa_mel_stream_*: live streams on this plan
};

using namespace fa;

FA_API void fa_mel_default_config(fa_mel_config *cfg) {
    if (!cfg) return;
    cfg->sample_rate = 16000;
    cfg->n_mels = 128;
    cfg->n_fft = 512;
    cfg->hop_length = 160;
    cfg->win_length = 400;
    cfg->preemph = 0.97f;
    cfg->pad_to = 0;
    cfg->log_floor = ldexpf(1.0f, -24);
    cfg->log_floor_mode = 0;
    cfg->window_periodic = 0;
}

static mel::MelConfig mel_config_of(const fa_mel_config *cfg) {
    return mel::MelConfig{cfg->sample_rate, cfg->n_mels,  cfg->n_fft,     cfg->hop_length,     cfg->win_length,
                          cfg->preemph,     cfg->pad_to,  cfg->log_floor, cfg->log_floor_mode, cfg->window_periodic};
}

static int create_mel(const mel::MelConfig &c, fa_mel **out) {
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    std::unique_ptr<fa_mel> h(new fa_mel());
    const int st = h->plan.init(c);
    if (st != FA_OK) return st;
    *out = h.release();
    return FA_STATUS_OK;
}

FA_API fa_status fa_mel_create(const fa_mel_config *cfg, fa_mel **out) {
    return guard(__func__, [&]() -> int {
        if (!cfg || !out) return FA_STATUS_INVALID_ARGUMENT;
        *out = nullptr;
        return create_mel(mel_config_of(cfg), out);
    });
}

FA_API void fa_mel_ex_default_config(fa_mel_ex_config *cfg) {
    if (!cfg) return;
    fa_mel_default_config(&cfg->base);
    cfg->filterbank = FA_MEL_FB_AUDIO_MEL;
    cfg->filter_sample_rate = 0;
    cfg->f_min = 0.0f;
    cfg->f_max = 0.0f;
    cfg->center_edge = FA_MEL_EDGE_ZERO;
    cfg->spectrum_power = 2.0f;
    cfg->log_mean = 0.0f;
    cfg->log_std = 1.0f;
}

// CohereMelSpectrogram.Config() (CoherePipeline.swift:55-77) with CohereAsrConfig.MelSpec: nFFT = nextPow2(winLength)
FA_API void fa_mel_preset_cohere(fa_mel_ex_config *cfg) {
    if (!cfg) return;
    fa_mel_ex_default_config(cfg);
    fa_mel_config &b = cfg->base;
    b.sample_rate = 16000;
    b.win_length = 400;
    b.hop_length = 160;
    b.n_mels = 128;
    b.n_fft = 1;
    while (b.n_fft < b.win_length) b.n_fft <<= 1;   // nextPowerOfTwo(atLeast:) (:265-269): 512
    b.preemph = 0.97f;
    b.log_floor = 5.9604645e-08f;   // logZeroGuard 2^-24, additive
    b.log_floor_mode = 0;
    b.window_periodic = 0;
    cfg->filterbank = FA_MEL_FB_COHERE;
    cfg->f_min = 0.0f;
    cfg->f_max = 8000.0f;
}

// StyleTTS2Constants (StyleTTS2Constants.swift:13, :43-52): 24 kHz audio, the table built for 16 kHz
FA_API void fa_mel_preset_styletts2(fa_mel_ex_config *cfg) {
    if (!cfg) return;
    fa_mel_ex_default_config(cfg);
    fa_mel_config &b = cfg->base;
    b.sample_rate = 24000;
    b.n_fft = 2048;
    b.win_length = 1200;
    b.hop_length = 300;
    b.n_mels = 80;
    b.preemph = 0.0f;
    b.log_floor = 1e-5f;
    b.log_floor_mode = 0;
    b.window_periodic = 1;
    cfg->filterbank = FA_MEL_FB_STYLETTS2;
    cfg->filter_sample_rate = 16000;
    cfg->center_edge = FA_MEL_EDGE_REFLECT;
    cfg->log_mean = -4.0f;
    cfg->log_std = 4.0f;
}

// LuxTtsConstants (LuxTtsConstants.swift:11-21): torchaudio MelSpectrogram(24000, 1024, hop 256, 100 mels, power 1)
FA_API void fa_mel_preset_luxtts(fa_mel_ex_config *cfg) {
    if (!cfg) return;
    fa_mel_ex_default_config(cfg);
    fa_mel_config &b = cfg->base;
    b.sample_rate = 24000;
    b.n_fft = 1024;
    b.win_length = 1024;
    b.hop_length = 256;
    b.n_mels = 100;
    b.preemph = 0.0f;
    b.log_floor = 1e-7f;
    b.log_floor_mode = 1;
    b.window_periodic = 1;
    cfg->filterbank = FA_MEL_FB_LUXTTS;
    cfg->center_edge = FA_MEL_EDGE_REFLECT;
    cfg->spectrum_power = 1.0f;
}

FA_API fa_status fa_mel_create_ex(const fa_mel_ex_config *cfg, fa_mel **out) {
    return guard(__func__, [&]() -> int {
        if (!cfg || !out) return FA_STATUS_INVALID_ARGUMENT;
        *out = nullptr;
        mel::MelConfig c = mel_config_of(&cfg->base);
        c.fb_kind = cfg->filterbank;
        c.filter_sample_rate = cfg->filter_sample_rate;
        c.f_min = cfg->f_min;
        c.f_max = cfg->f_max;
        c.center_edge = cfg->center_edge;
        c.spectrum_power = cfg->spectrum_power;
        c.log_mean = cfg->log_mean;
        c.log_std = cfg->log_std;
        if (const char *why = mel::check_ex_config(c))   // before the device is touched
            return refuse("mel ex config: %s", why);
        return create_mel(c, out);
    });
}

FA_API void fa_mel_destroy(fa_mel *mel) { delete mel; }

FA_API fa_status fa_mel_get_window(const fa_mel *mel, float *out, size_t len) {
    return guard(__func__, [&]() -> int {
        if (!mel || !out) return FA_STATUS_INVALID_ARGUMENT;
        const auto &w = mel->plan.window;
        if (len < w.size()) return FA_STATUS_OUTPUT_TOO_SMALL;
        std::memcpy(out, w.data(), w.size() * sizeof(float));
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_mel_get_filterbank(const fa_mel *mel, float *out, size_t len) {
    return guard(__func__, [&]() -> int {
        if (!mel || !out) return FA_STATUS_INVALID_ARGUMENT;
        const auto &f = mel->plan.filterbank;
        if (len < f.size()) return FA_STATUS_OUTPUT_TOO_SMALL;
        std::memcpy(out, f.data(), f.size() * sizeof(float));
        return FA_STATUS_OK;
    });
}

FA_API int64_t fa_mel_frame_count(const fa_mel *mel, int64_t n, int32_t padding_mode, int64_t expected) {
    if (!mel) {
        fa::set_error("fa_mel_frame_count: mel is NULL");
        return -1;
    }
    return mel->plan.frame_count(n, padding_mode, expected);
}

FA_API fa_status fa_mel_set_precision(fa_mel *mel, int32_t precision) {
    return guard(__func__, [&]() -> int {
        if (!mel || (precision != FA_MEL_PRECISION_F64 && precision != FA_MEL_PRECISION_F32))
            return refuse("precision must be FA_MEL_PRECISION_F64 (0) or FA_MEL_PRECISION_F32 (1)");
        mel->plan.precision = precision;
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_mel_set_pipeline_chunks(fa_mel *mel, int32_t chunks) {
    return guard(__func__, [&]() -> int {
        if (!mel || chunks < 1 || chunks > 1024) return FA_STATUS_INVALID_ARGUMENT;
        mel->plan.pipeline_chunks = chunks;
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_mel_set_zero_copy_output(fa_mel *mel, int32_t enabled) {
    return guard(__func__, [&]() -> int {
        if (!mel) return FA_STATUS_INVALID_ARGUMENT;
        mel->plan.zero_copy_out = enabled != 0;
        return FA_STATUS_OK;
    });
}
FA_API int32_t fa_mel_get_precision(const fa_mel *mel) {
    if (!mel) {
        fa::set_error("fa_mel_get_precision: mel is NULL");
        return -1;
    }
    return mel->plan.precision;
}

static bool mel_args_ok(int32_t mode, int32_t layout) {
    if (mode < FA_MEL_PAD_CENTER || mode > FA_MEL_LEGACY_COMPUTE || layout < FA_MEL_TIME_MAJOR || layout > FA_MEL_MEL_MAJOR) {
        fa::set_error("padding_mode must be 0..2 and layout 0..1");
        return false;
    }
    return true;
}

FA_API fa_status fa_mel_compute(fa_mel *mel, const float *audio, size_t n, float last, int32_t mode, int64_t expected,
                                int32_t layout, float *out, size_t out_len, int64_t *mel_length, int64_t *num_frames) {
    return guard(__func__, [&]() -> int {
        if (!mel || !out || (!audio && n) || !mel_args_ok(mode, layout)) return FA_STATUS_INVALID_ARGUMENT;
        long long ml = 0, nf = 0;
        const double rate = mel->plan.cfg.sample_rate;
        const resample::AudioFormat mono_f32{rate, rate, 1, resample::kPcmF32, 1, resample::kAlgoAuto};
        const int st = mel->plan.compute_host(audio, (long long)n, mono_f32, last, mode, expected, layout, out,
                                              capacity(out_len), &ml, &nf, nullptr);
        if (mel_length) *mel_length = ml;
        if (num_frames) *num_frames = nf;
        return st;
    });
}

FA_API fa_status fa_audio_to_mel(fa_mel *mel, const void *pcm, int64_t frames, const fa_audio_format *fmt, float last,
                                 int32_t mode, int32_t layout, float *out, size_t out_len, int64_t *mel_length,
                                 int64_t *num_frames, int64_t *resampled_count) {
    return guard(__func__, [&]() -> int {
        if (!mel || !out || frames < 0 || (!pcm && frames) || !resample::audio_format_ok(fmt) ||
            !mel_args_ok(mode, layout))
            return FA_STATUS_INVALID_ARGUMENT;
        if (fmt->out_rate != (double)mel->plan.cfg.sample_rate)
            return refuse("fa_audio_to_mel: out_rate %.3f differs from the handle's sample_rate %d", fmt->out_rate,
                          mel->plan.cfg.sample_rate);
        long long ml = 0, nf = 0, rs = 0;
        const int st = mel->plan.compute_host(pcm, (long long)frames, resample::to_format(fmt), last, mode, -1, layout,
                                              out, capacity(out_len), &ml, &nf, &rs);
        if (mel_length) *mel_length = ml;
        if (num_frames) *num_frames = nf;
        if (resampled_count) *resampled_count = rs;
        return st;
    });
}

FA_API fa_status fa_mel_compute_device(fa_mel *mel, const float *d_audio, size_t n, float last, int32_t mode,
                                       int64_t expected, int32_t layout, float *d_out, size_t out_len,
                                       int64_t *mel_length, int64_t *num_frames) {
    return guard(__func__, [&]() -> int {
        if (!mel || !d_out || (!d_audio && n) || !mel_args_ok(mode, layout)) return FA_STATUS_INVALID_ARGUMENT;
        long long ml = 0, nf = 0;
        const int st = mel->plan.compute_device(d_audio, (long long)n, last, mode, expected, layout, d_out,
                                                capacity(out_len), &ml, &nf, mel->plan.streams[1]);
        if (mel_length) *mel_length = ml;
        if (num_frames) *num_frames = nf;
        return st;
    });
}

FA_API fa_status fa_mel_compute_batch(fa_mel *mel, const float *audio, const int64_t *offsets, int32_t count,
                                      const float *last, int32_t mode, int32_t layout, float *out,
                                      const int64_t *out_offsets, int64_t *mel_lengths, int64_t *num_frames) {
    return guard(__func__, [&]() -> int {
        if (!mel || !audio || !offsets || !out || !out_offsets || count < 0 || !mel_args_ok(mode, layout))
            return FA_STATUS_INVALID_ARGUMENT;
        return mel->plan.compute_batch_host(audio, offsets, count, last, mode, layout, out, out_offsets, mel_lengths,
                                            num_frames);
    });
}

FA_API fa_status fa_mel_compute_batch_device(fa_mel *mel, const float *d_audio, const int64_t *offsets, int32_t count,
                                             const float *last, int32_t mode, int32_t layout, float *d_out,
                                             const int64_t *out_offsets, int64_t *mel_lengths, int64_t *num_frames) {
    return guard(__func__, [&]() -> int {
        if (!mel || !d_audio || !offsets || !d_out || !out_offsets || count < 0 || !mel_args_ok(mode, layout))
            return FA_STATUS_INVALID_ARGUMENT;
        return mel->plan.compute_batch_device(d_audio, offsets, count, last, mode, layout, d_out, out_offsets,
                                              mel_lengths, num_frames, mel->plan.streams[1]);
    });
}

FA_API fa_status fa_mel_timer_start(fa_mel *mel) {
    return guard(__func__, [&]() -> int {
        if (!mel) return FA_STATUS_INVALID_ARGUMENT;
        return mel->plan.timer_start();
    });
}
FA_API fa_status fa_mel_timer_stop_ms(fa_mel *mel, float *elapsed_ms) {
    return guard(__func__, [&]() -> int {
        if (!mel || !elapsed_ms) return FA_STATUS_INVALID_ARGUMENT;
        return mel->plan.timer_stop_ms(elapsed_ms);
    });
}

// Live streams (SortformerDiarizer.swift:204-217, :417-424, :842-901): sessions on the handle, see mel_stream.cu.
FA_API fa_status fa_mel_stream_open(fa_mel *mel, int32_t *session) {
    return guard(__func__, [&]() -> int {
        if (!mel || !session) return FA_STATUS_INVALID_ARGUMENT;
        int id = -1;
        const int st = mel->sessions.open(mel->plan, &id);
        if (st == FA_OK) *session = id;
        return st;
    });
}

FA_API fa_status fa_mel_stream_close(fa_mel *mel, int32_t session) {
    return guard(__func__, [&]() -> int {
        if (!mel) return FA_STATUS_INVALID_ARGUMENT;
        return mel->sessions.close(session);
    });
}

FA_API int64_t fa_mel_stream_frames(const fa_mel *mel, int32_t session, int64_t new_samples, int32_t finish) {
    const long long frames = mel ? mel->sessions.frames(mel->plan, session, new_samples, finish != 0) : -1;
    if (frames < 0) fa::set_error("fa_mel_stream_frames: mel is NULL, session %d is not open or new_samples < 0", session);
    return frames;
}

static int mel_stream_push(fa_mel *mel, int32_t count, const int32_t *sessions, const float *audio,
                           const int64_t *offsets, const int32_t *finish, bool device, float *out, size_t out_len,
                           int64_t *frames) {
    if (!mel) return FA_STATUS_INVALID_ARGUMENT;
    return mel->sessions.push(mel->plan, count, sessions, audio, offsets, finish, device, out, capacity(out_len), frames);
}

FA_API fa_status fa_mel_stream_push(fa_mel *mel, int32_t count, const int32_t *sessions, const float *audio,
                                    const int64_t *offsets, const int32_t *finish, float *out, size_t out_len,
                                    int64_t *frames) {
    return guard(__func__,
                 [&] { return mel_stream_push(mel, count, sessions, audio, offsets, finish, false, out, out_len, frames); });
}

FA_API fa_status fa_mel_stream_push_device(fa_mel *mel, int32_t count, const int32_t *sessions, const float *d_audio,
                                           const int64_t *offsets, const int32_t *finish, float *d_out, size_t out_len,
                                           int64_t *frames) {
    return guard(__func__, [&] {
        return mel_stream_push(mel, count, sessions, d_audio, offsets, finish, true, d_out, out_len, frames);
    });
}

// UnifiedMelExtractor.features(window:validCount:) (UnifiedMelExtractor.swift:52-86): log-mel + per-feature
// normalisation + [1, nMels, T] packing, normalisation and packing as a device epilogue of the mel kernel.
FA_API fa_status fa_mel_unified_features(fa_mel *mel, const float *window, size_t window_samples, size_t valid_count,
                                         float *out, size_t out_len, int64_t *total_frames, int32_t *valid_frames) {
    return guard(__func__, [&]() -> int {
        if (!mel || !out || (!window && window_samples)) return FA_STATUS_INVALID_ARGUMENT;
        long long T = 0;
        int valid = 0;
        const int st = fa::mel::unified_features(mel->plan, window, (long long)window_samples, (long long)valid_count,
                                                 out, capacity(out_len), &T, &valid);
        if (total_frames) *total_frames = T;
        if (valid_frames) *valid_frames = valid;
        return st;
    });
}

// LSEENDPreprocessor.processAudioQueue (LSEENDPreprocessor.swift:249-283): .prePadded log-mel of one audio chunk,
// log10 scaling and cumulative mean normalisation; (cmn_mean, cmn_count) is the preprocessor's running state.
FA_API fa_status fa_mel_lseend_features(fa_mel *mel, const float *chunk, size_t n, float *cmn_mean, int64_t *cmn_count,
                                        float *out, size_t out_len, int64_t *frames) {
    return guard(__func__, [&]() -> int {
        if (!mel || !cmn_mean || !cmn_count || *cmn_count < 0 || (!chunk && n) || (!out && out_len))
            return FA_STATUS_INVALID_ARGUMENT;
        long long T = 0, count = *cmn_count;
        const int st =
            fa::mel::lseend_features(mel->plan, chunk, (long long)n, cmn_mean, &count, out, capacity(out_len), &T);
        *cmn_count = count;
        if (frames) *frames = T;
        return st;
    });
}

// CohereMelSpectrogram.compute + padOrTruncate (CoherePipeline.swift:127-263), StyleTTS2MelExtractor.compute
// (StyleTTS2MelExtractor.swift:77-141), LuxTtsMelExtractor.extract (LuxTtsMelExtractor.swift:52-132): mel_adapters.cu.
FA_API fa_status fa_mel_cohere_features(fa_mel *mel, const float *audio, size_t n, int64_t fixed_frames, float *out,
                                        size_t out_len, int64_t *frames, int64_t *valid_frames) {
    return guard(__func__, [&]() -> int {
        if (!mel || !out || (!audio && n)) return FA_STATUS_INVALID_ARGUMENT;
        long long W = 0, valid = 0;
        const int st = fa::mel::cohere_features(mel->plan, audio, (long long)n, (long long)fixed_frames, out,
                                                capacity(out_len), &W, &valid);
        if (frames) *frames = W;
        if (valid_frames) *valid_frames = valid;
        return st;
    });
}

FA_API fa_status fa_mel_styletts2_features(fa_mel *mel, const float *audio, size_t n, float *out, size_t out_len,
                                           int64_t *frames) {
    return guard(__func__, [&]() -> int {
        if (!mel || !out || (!audio && n)) return FA_STATUS_INVALID_ARGUMENT;
        long long T = 0;
        const int st = fa::mel::styletts2_features(mel->plan, audio, (long long)n, out, capacity(out_len), &T);
        if (frames) *frames = T;
        return st;
    });
}

FA_API fa_status fa_mel_luxtts_features(fa_mel *mel, const float *audio, size_t n, float *out, size_t out_len,
                                        int64_t *frames) {
    return guard(__func__, [&]() -> int {
        if (!mel || (!out && out_len) || (!audio && n)) return FA_STATUS_INVALID_ARGUMENT;
        long long T = 0;
        const int st = fa::mel::luxtts_features(mel->plan, audio, (long long)n, out, capacity(out_len), &T);
        if (frames) *frames = T;
        return st;
    });
}

// UnifiedMelExtractor.normalizePerFeature (UnifiedMelExtractor.swift:88-113).  O(T*M) on a caller-owned host
// buffer that is about to be handed to the encoder; not a GPU hot path.
FA_API fa_status fa_mel_normalize_per_feature(float *x, int64_t frames, int32_t n_mels, int64_t valid) {
    return guard(__func__, [&]() -> int {
        if (!x || frames < 0 || n_mels <= 0) return FA_STATUS_INVALID_ARGUMENT;
        if (valid > frames) valid = frames;   // UnifiedMelExtractor.swift:66: validFrames = min(validCount / hop, totalFrames)
        if (frames == 0) return FA_STATUS_OK;
        if (valid <= 0) {                     // no valid frame: everything is padding
            std::memset(x, 0, sizeof(float) * (size_t)frames * n_mels);
            return FA_STATUS_OK;
        }
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) {
            return mel::normalize_per_feature_host(C, x, (long long)frames, n_mels, (long long)valid);
        });
    });
}
