// C ABI of libfluidaudio_b200.so (declared in include/fluidaudio_b200.h and include/FastClusterWrapper.h).
// No exception and no CUDA type crosses this boundary; there is no CPU fallback behind it.  Every entry point that
// returns a status returns through guard() (c_abi.h).
#include "../../include/FastClusterWrapper.h"
#include "c_abi.h"

#include "ahc_plan.h"
#include "assign_host.h"
#include "call_context.h"
#include "cluster_plan.h"
#include "mel_plan.h"
#include "kmeans_plan.h"
#include "prepare_plan.h"
#include "reconstruct_host.h"
#include "sortformer_plan.h"
#include "timeline_plan.h"

#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

// The opaque handles of the header.
struct fa_mel {
    fa::mel::MelPlan plan;
    fa::mel::MelStreamSet sessions;   // fa_mel_stream_*: live streams on this plan
};
struct fa_sortformer {
    fa::sortformer::SortformerSet set;
};
struct fa_diarizer_timeline {
    fa::timeline::TimelineSet set;
};

namespace fa {

// The last failure's text on this thread, and how many times it has been set (error_serial).
struct ErrorText {
    char text[512];
    unsigned serial;
};
static thread_local ErrorText g_error{};
void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error.text, sizeof(g_error.text), fmt, ap);
    va_end(ap);
    ++g_error.serial;
}
const char *last_error() { return g_error.text; }
unsigned error_serial() { return g_error.serial; }

const char *status_name(int status) {
    switch (status) {
    case FA_OK: return "FA_STATUS_OK";
    case FA_INVALID_ARGUMENT: return "FA_STATUS_INVALID_ARGUMENT";
    case FA_INDEX_OVERFLOW: return "FA_STATUS_INDEX_OVERFLOW";
    case FA_OUTPUT_TOO_SMALL: return "FA_STATUS_OUTPUT_TOO_SMALL";
    case FA_ALLOCATION_FAILURE: return "FA_STATUS_ALLOCATION_FAILURE";
    case FA_RUNTIME_ERROR: return "FA_STATUS_RUNTIME_ERROR";
    case FA_NO_DEVICE: return "FA_STATUS_NO_DEVICE";
    case FA_CUDA_ERROR: return "FA_STATUS_CUDA_ERROR";
    case FA_UNSUPPORTED: return "FA_STATUS_UNSUPPORTED";
    default: return "FA_STATUS_UNKNOWN_ERROR";
    }
}

std::atomic<long long> g_launches{0};

static int usable_device_count() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    int ok = 0;
    for (int i = 0; i < n; ++i) {
        cudaDeviceProp p;
        if (sm90_device_props(i, p) == FA_OK) ++ok;
    }
    return ok;
}

int require_device() {
    static std::atomic<int> cached{-1};
    int c = cached.load();
    if (c < 0) {
        c = usable_device_count();
        cached.store(c);
    }
    if (c <= 0) {
        set_error("no sm_90a (H100) device visible; fluidaudio_b200 has no CPU fallback");
        return FA_NO_DEVICE;
    }
    return FA_OK;
}

// timer state for fa_timer_*, per thread
static thread_local Event t_ev[2];

// Creates both timer events, or neither: a failed creation leaves the timer unset, so the next start tries again.
static int create_timer(Event (&ev)[2]) {
    int st = ev[0].create();
    if (st == FA_OK) st = ev[1].create();
    if (st != FA_OK) ev[0].reset();
    return st;
}

} // namespace fa

using namespace fa;

// ------------------------------------------------------------------------------------------------ runtime
FA_API const char *fa_version(void) { return "fluidaudio_b200 0.1.0 (sm_90a)"; }
FA_API const char *fa_last_error(void) { return fa::last_error(); }
FA_API int32_t fa_device_count(void) { return usable_device_count(); }

FA_API fa_status fa_set_device(int32_t ordinal) {
    return guard(__func__, [&]() -> int {
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        FA_CUDA_TRY(cudaSetDevice(ordinal));
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_device_synchronize(void) {
    return guard(__func__, [&]() -> int {
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        FA_CUDA_TRY(cudaDeviceSynchronize());
        return FA_STATUS_OK;
    });
}

FA_API int64_t fa_kernel_launch_count(void) { return g_launches.load(); }

FA_API fa_status fa_host_alloc(size_t bytes, void **out) {
    return guard(__func__, [&]() -> int {
        if (!out) return FA_STATUS_INVALID_ARGUMENT;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        FA_CUDA_TRY(cudaMallocHost(out, bytes ? bytes : 1));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_host_free(void *p) {
    return guard(__func__, [&]() -> int {
        if (p) FA_CUDA_TRY(cudaFreeHost(p));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_device_alloc(size_t bytes, void **out) {
    return guard(__func__, [&]() -> int {
        if (!out) return FA_STATUS_INVALID_ARGUMENT;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        FA_CUDA_TRY(cudaMalloc(out, bytes ? bytes : 1));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_device_free(void *p) {
    return guard(__func__, [&]() -> int {
        if (p) FA_CUDA_TRY(cudaFree(p));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_memcpy_h2d(void *dst, const void *src, size_t bytes) {
    return guard(__func__, [&]() -> int {
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        FA_CUDA_TRY(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_memcpy_d2h(void *dst, const void *src, size_t bytes) {
    return guard(__func__, [&]() -> int {
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        FA_CUDA_TRY(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
        return FA_STATUS_OK;
    });
}

// Bare copy-engine probe: `reps` rounds of an H2D copy of h2d_bytes and a D2H copy of d2h_bytes issued together on two
// streams (device scratch allocated here), wall-clock per round.  bench.py uses it to name the floor under every
// host-buffer (end-to-end) number: what the PCIe / host-memory path delivers with no kernel in the way.
FA_API fa_status fa_memcpy_probe(const void *host_src, size_t h2d_bytes, void *host_dst, size_t d2h_bytes, int32_t reps,
                                 float *ms_per_round) {
    return guard(__func__, [&]() -> int {
        if (!ms_per_round || reps < 1 || (!host_src && h2d_bytes) || (!host_dst && d2h_bytes))
            return FA_STATUS_INVALID_ARGUMENT;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        Stream s[2];
        DeviceBuffer<> a, b;
        int st = a.grow(h2d_bytes + 16);
        if (st == FA_OK) st = b.grow(d2h_bytes + 16);
        if (st != FA_OK) return st;
        FA_CUDA_TRY(cudaMemset(b.data(), 0, d2h_bytes + 16));
        for (auto &x : s)
            if (st == FA_OK) st = x.create();
        if (st != FA_OK) return st;
        FA_CUDA_TRY(cudaDeviceSynchronize());
        const auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < reps; ++i) {
            if (h2d_bytes) FA_CUDA_TRY(cudaMemcpyAsync(a.data(), host_src, h2d_bytes, cudaMemcpyHostToDevice, s[0]));
            if (d2h_bytes) FA_CUDA_TRY(cudaMemcpyAsync(host_dst, b.data(), d2h_bytes, cudaMemcpyDeviceToHost, s[1]));
            FA_CUDA_TRY(cudaStreamSynchronize(s[0]));
            FA_CUDA_TRY(cudaStreamSynchronize(s[1]));
        }
        const auto t1 = std::chrono::steady_clock::now();
        *ms_per_round = (float)(std::chrono::duration<double, std::milli>(t1 - t0).count() / reps);
        return FA_STATUS_OK;
    });
}

// Events on the legacy default stream order against every blocking stream AND, because the library's own streams
// are non-blocking, the timed entry points synchronise their streams before returning (device-side async calls
// are timed by the caller bracketing fa_device_synchronize()).
FA_API fa_status fa_timer_start(void) {
    return guard(__func__, [&]() -> int {
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        if (!t_ev[0]) {
            const int st = create_timer(t_ev);
            if (st != FA_OK) return st;
        }
        FA_CUDA_TRY(cudaDeviceSynchronize());
        FA_CUDA_TRY(cudaEventRecord(t_ev[0], 0));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_timer_stop_ms(float *elapsed_ms) {
    return guard(__func__, [&]() -> int {
        if (!elapsed_ms || !t_ev[0]) return FA_STATUS_INVALID_ARGUMENT;
        FA_CUDA_TRY(cudaDeviceSynchronize());
        FA_CUDA_TRY(cudaEventRecord(t_ev[1], 0));
        FA_CUDA_TRY(cudaEventSynchronize(t_ev[1]));
        FA_CUDA_TRY(cudaEventElapsedTime(elapsed_ms, t_ev[0], t_ev[1]));
        return FA_STATUS_OK;
    });
}

// ------------------------------------------------------------------------------------------------ mel
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
        if (const char *why = mel::check_ex_config(c)) {   // before the device is touched
            fa::set_error("mel ex config: %s", why);
            return FA_STATUS_INVALID_ARGUMENT;
        }
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
        if (!mel || (precision != FA_MEL_PRECISION_F64 && precision != FA_MEL_PRECISION_F32)) {
            fa::set_error("precision must be FA_MEL_PRECISION_F64 (0) or FA_MEL_PRECISION_F32 (1)");
            return FA_STATUS_INVALID_ARGUMENT;
        }
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

// CUDA-event timing on the stream the mel kernels are launched on (device-resident entry points are asynchronous).
FA_API fa_status fa_mel_timer_start(fa_mel *mel) {
    return guard(__func__, [&]() -> int {
        if (!mel) return FA_STATUS_INVALID_ARGUMENT;
        if (!mel->plan.timer[0]) {
            const int st = create_timer(mel->plan.timer);
            if (st != FA_OK) return st;
        }
        FA_CUDA_TRY(cudaStreamSynchronize(mel->plan.streams[1]));
        FA_CUDA_TRY(cudaEventRecord(mel->plan.timer[0], mel->plan.streams[1]));
        return FA_STATUS_OK;
    });
}
FA_API fa_status fa_mel_timer_stop_ms(fa_mel *mel, float *elapsed_ms) {
    return guard(__func__, [&]() -> int {
        if (!mel || !elapsed_ms) return FA_STATUS_INVALID_ARGUMENT;
        if (!mel->plan.timer[0]) return FA_STATUS_INVALID_ARGUMENT;
        FA_CUDA_TRY(cudaEventRecord(mel->plan.timer[1], mel->plan.streams[1]));
        FA_CUDA_TRY(cudaEventSynchronize(mel->plan.timer[1]));
        FA_CUDA_TRY(cudaEventElapsedTime(elapsed_ms, mel->plan.timer[0], mel->plan.timer[1]));
        return FA_STATUS_OK;
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

// ------------------------------------------------------------------------------------------------ AudioConverter stage
static bool audio_format_ok(const fa_audio_format *f) {
    if (!f || !(f->in_rate > 0) || !(f->out_rate > 0) || f->channels < 1 || f->channels > 64 ||
        (f->format != FA_PCM_F32 && f->format != FA_PCM_I16) || f->algorithm < 0 || f->algorithm > 2) {
        fa::set_error("audio format: rates must be positive, 1..64 channels, format F32/I16, algorithm 0..2");
        return false;
    }
    return true;
}
static resample::AudioFormat to_format(const fa_audio_format *f) {
    return resample::AudioFormat{f->in_rate, f->out_rate, f->channels, f->format, f->interleaved ? 1 : 0, f->algorithm};
}

FA_API int64_t fa_resample_output_count(const fa_audio_format *fmt, int64_t frames) {
    if (!fmt || frames < 0 || !(fmt->in_rate > 0) || !(fmt->out_rate > 0)) {
        fa::set_error("fa_resample_output_count: fmt is NULL, frames < 0 or a rate is not positive");
        return -1;
    }
    return resample::output_count(frames, fmt->in_rate, fmt->out_rate);
}

static int audio_resample(const void *pcm, int64_t frames, const fa_audio_format *fmt, float *out, int64_t out_cap,
                          int64_t *out_count) {
    if (!audio_format_ok(fmt) || frames < 0 || !out_count) return FA_STATUS_INVALID_ARGUMENT;
    const long long n = resample::output_count(frames, fmt->in_rate, fmt->out_rate);
    *out_count = n;
    if (!out) return FA_STATUS_OK;            // sizing call: pcm may be NULL
    if (!pcm && frames) {
        fa::set_error("fa_audio_resample: pcm is NULL");
        return FA_STATUS_INVALID_ARGUMENT;
    }
    if (out_cap < n) return FA_STATUS_OUTPUT_TOO_SMALL;
    if (n == 0) return FA_STATUS_OK;
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    const resample::AudioFormat f = to_format(fmt);
    resample::Design d;
    if (f.in_rate != f.out_rate) {
        const int st = resample::make_design(f.in_rate, f.out_rate, d);
        if (st != FA_OK) return st;
    }
    const size_t bytes = (size_t)frames * f.channels * (f.format == resample::kPcmI16 ? 2 : 4);
    return with_context(0, [&](CallContext &C) -> int {
        HostStaging H(true, C.stream);
        const char *d_pcm;
        const float *d_tab;
        float *d_out;
        int st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
            d_pcm = l.in(static_cast<const char *>(pcm), bytes, 16);
            d_tab = l.in(d.table.empty() ? nullptr : d.table.data(), d.table.size());
            d_out = l.out(out, (size_t)n);
        });
        if (st != FA_OK) return st;
        st = resample::launch_convert(d_pcm, frames, f, d, d_tab, d_out, 0, n, C.stream);
        if (st != FA_OK) return st;
        FA_CUDA_TRY(H.finish());
        return FA_OK;
    });
}

FA_API fa_status fa_audio_resample(const void *pcm, int64_t frames, const fa_audio_format *fmt, float *out,
                                   int64_t out_cap, int64_t *out_count) {
    return guard(__func__, [&] { return audio_resample(pcm, frames, fmt, out, out_cap, out_count); });
}

FA_API fa_status fa_audio_to_mel(fa_mel *mel, const void *pcm, int64_t frames, const fa_audio_format *fmt, float last,
                                 int32_t mode, int32_t layout, float *out, size_t out_len, int64_t *mel_length,
                                 int64_t *num_frames, int64_t *resampled_count) {
    return guard(__func__, [&]() -> int {
        if (!mel || !out || frames < 0 || (!pcm && frames) || !audio_format_ok(fmt) || !mel_args_ok(mode, layout))
            return FA_STATUS_INVALID_ARGUMENT;
        if (fmt->out_rate != (double)mel->plan.cfg.sample_rate) {
            fa::set_error("fa_audio_to_mel: out_rate %.3f differs from the handle's sample_rate %d", fmt->out_rate,
                          mel->plan.cfg.sample_rate);
            return FA_STATUS_INVALID_ARGUMENT;
        }
        long long ml = 0, nf = 0, rs = 0;
        const int st = mel->plan.compute_host(pcm, (long long)frames, to_format(fmt), last, mode, -1, layout, out,
                                              capacity(out_len), &ml, &nf, &rs);
        if (mel_length) *mel_length = ml;
        if (num_frames) *num_frames = nf;
        if (resampled_count) *resampled_count = rs;
        return st;
    });
}

// AudioConverter.linearResample (AudioConverter.swift:388-442): boundary glue for >2-channel input.
FA_API fa_status fa_linear_resample(const float *in, int64_t frames, int32_t channels, double in_rate, double out_rate,
                                    float *out, int64_t out_cap, int64_t *out_count) {
    return guard(__func__, [&]() -> int {
        if (frames < 0 || channels <= 0 || !(in_rate > 0) || !(out_rate > 0) || !out_count || (out && !in && frames))
            return FA_STATUS_INVALID_ARGUMENT;
        // planar float32, the two-tap float32 interpolation whatever the channel count: the converter stage's linear kernel
        fa_audio_format fmt{};
        fmt.in_rate = in_rate;
        fmt.out_rate = out_rate;
        fmt.channels = channels;
        fmt.format = FA_PCM_F32;
        fmt.interleaved = 0;
        fmt.algorithm = FA_RESAMPLE_LINEAR;
        return audio_resample(in, frames, &fmt, out, out_cap, out_count);
    });
}

// ------------------------------------------------------------------------------------------------ clustering
static fastcluster_wrapper_status to_fc(int st) {
    switch (st) {
    case FA_OK: return FASTCLUSTER_WRAPPER_SUCCESS;
    case FA_INVALID_ARGUMENT: return FASTCLUSTER_WRAPPER_INVALID_ARGUMENT;
    case FA_INDEX_OVERFLOW: return FASTCLUSTER_WRAPPER_INDEX_OVERFLOW;
    case FA_OUTPUT_TOO_SMALL: return FASTCLUSTER_WRAPPER_OUTPUT_TOO_SMALL;
    case FA_ALLOCATION_FAILURE: return FASTCLUSTER_WRAPPER_ALLOCATION_FAILURE;
    case FA_UNKNOWN_ERROR: return FASTCLUSTER_WRAPPER_UNKNOWN_ERROR;
    default: return FASTCLUSTER_WRAPPER_RUNTIME_ERROR;   // NaN, CUDA failure, no device, unsupported size
    }
}

FA_API fastcluster_wrapper_status fastcluster_compute_centroid_linkage(const double *data, size_t pointCount,
                                                                       size_t dimension, double *dendrogramOut,
                                                                       size_t dendrogramLength) {
    return to_fc(guard(__func__, [&]() -> int {
        // argument contract first, exactly as FastClusterWrapper.cpp:203-223 (no device needed for these)
        if (data == nullptr || dendrogramOut == nullptr) return FA_INVALID_ARGUMENT;
        if (pointCount == 0) return FA_OK;
        if (dimension == 0) return FA_INVALID_ARGUMENT;
        if (pointCount > 0x7fffffffull || dimension > 0x7fffffffull) return FA_INDEX_OVERFLOW;
        const size_t need = pointCount > 1 ? (pointCount - 1) * 4 : 0;
        if (dendrogramLength < need) return FA_OUTPUT_TOO_SMALL;
        if (pointCount == 1) return FA_OK;
        if (require_device() != FA_OK) return FA_NO_DEVICE;
        return with_context(0, [&](CallContext &C) {
            return C.solver.linkage_host(data, pointCount, dimension, dendrogramOut, dendrogramLength);
        });
    }));
}

FA_API void fa_ahc_last_stage_ms(float *out4) {
    if (!out4) return;
    const float *m = ahc::last_stage_ms();
    for (int q = 0; q < 4; ++q) out4[q] = m[q];
}

FA_API fa_status fa_l2_normalize_rows(const double *x, size_t rows, size_t dim, double *out) {
    return guard(__func__, [&]() -> int {
        if (!x || !out) return FA_STATUS_INVALID_ARGUMENT;
        if (rows == 0 || dim == 0) return FA_STATUS_OK;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) { return l2_normalize_rows(C, x, rows, dim, out); });
    });
}

FA_API fa_status fa_dendrogram_cut(const double *Z, size_t count, double threshold, int32_t *labels) {
    return guard(__func__, [&]() -> int {
        if ((!Z && count > 1) || (!labels && count > 0)) return FA_STATUS_INVALID_ARGUMENT;
        ahc::dendrogram_cut(Z, (long long)count, threshold, labels);
        return FA_STATUS_OK;
    });
}

// AHCClustering.cluster (AHCClustering.swift:20-67)
FA_API fa_status fa_ahc_cluster(const double *features, size_t count, size_t dim, double threshold, int32_t *labels) {
    return guard(__func__, [&]() -> int {
        if (count == 0) return FA_STATUS_OK;                       // guard count > 0 else []
        if (!labels) return FA_STATUS_INVALID_ARGUMENT;
        if (dim == 0) {                                            // zero-dimension vectors: all cluster 0 (:26-28)
            for (size_t i = 0; i < count; ++i) labels[i] = 0;
            return FA_STATUS_OK;
        }
        if (!features) return FA_STATUS_INVALID_ARGUMENT;
        if (count == 1) {
            labels[0] = 0;
            return FA_STATUS_OK;
        }
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) { return ahc_cluster(C, features, count, dim, threshold, labels); });
    });
}

FA_API void fa_vbx_default_config(fa_vbx_config *cfg) {
    if (!cfg) return;
    cfg->Fa = 0.07;
    cfg->Fb = 0.8;
    cfg->max_iterations = 20;
    cfg->epsilon = 1e-4;
    cfg->init_smoothing = 7.0;
}

FA_API void fa_cluster_default_config(fa_cluster_config *cfg) {
    if (!cfg) return;
    cfg->threshold = 0.6;
    fa_vbx_default_config(&cfg->vbx);
    cfg->num_speakers = cfg->min_speakers = cfg->max_speakers = FA_NO_VALUE;
    cfg->reserved = 0;
}

FA_API void fa_reconstruct_default_config(fa_reconstruct_config *cfg) {
    if (!cfg) return;
    const reconstruct::Config d;
    cfg->frame_duration = d.frame_duration;
    cfg->window_duration = d.window_duration;
    cfg->min_gap_duration = d.min_gap_duration;
    cfg->seg_min_duration_off = d.seg_min_duration_off;
    cfg->seg_min_duration_on = d.seg_min_duration_on;
    cfg->min_segment_duration = d.min_segment_duration;
    cfg->exclusive_segments = d.exclusive_segments ? 1 : 0;
    cfg->reserved = 0;
}

FA_API fa_status fa_build_segments(const float *weights, int32_t num_chunks, int32_t num_frames, int32_t num_speakers,
                                   const double *chunk_offsets, int32_t offsets_count, const int32_t *hard_clusters,
                                   int32_t hard_rows, int32_t centroid_count, const fa_reconstruct_config *cfg,
                                   int32_t *seg_cluster, float *seg_start, float *seg_end, float *seg_quality,
                                   int32_t segment_cap, int32_t *segment_count) {
    return guard(__func__, [&]() -> int {
        if (!cfg || !segment_count || num_speakers < 0 || offsets_count < 0 || hard_rows < 0 || segment_cap < 0 ||
            (num_chunks > 0 && num_frames > 0 && num_speakers > 0 && !weights) || (offsets_count > 0 && !chunk_offsets) ||
            (hard_rows > 0 && !hard_clusters))
            return FA_STATUS_INVALID_ARGUMENT;
        reconstruct::Config c;
        c.frame_duration = cfg->frame_duration;
        c.window_duration = cfg->window_duration;
        c.min_gap_duration = cfg->min_gap_duration;
        c.seg_min_duration_off = cfg->seg_min_duration_off;
        c.seg_min_duration_on = cfg->seg_min_duration_on;
        c.min_segment_duration = cfg->min_segment_duration;
        c.exclusive_segments = cfg->exclusive_segments != 0;
        std::vector<reconstruct::Segment> segs;
        reconstruct::build_segments(weights, num_chunks, num_frames, num_speakers, chunk_offsets, offsets_count,
                                    hard_clusters, hard_rows, centroid_count, c, segs);
        *segment_count = (int32_t)segs.size();
        const int32_t n = std::min<int32_t>((int32_t)segs.size(), segment_cap);
        for (int32_t i = 0; i < n; ++i) {
            if (seg_cluster) seg_cluster[i] = segs[i].cluster;
            if (seg_start) seg_start[i] = segs[i].start;
            if (seg_end) seg_end[i] = segs[i].end;
            if (seg_quality) seg_quality[i] = segs[i].quality;
        }
        return (int32_t)segs.size() > segment_cap ? FA_STATUS_OUTPUT_TOO_SMALL : FA_STATUS_OK;
    });
}

FA_API fa_status fa_build_speaker_database(const int32_t *seg_cluster, int32_t segment_count, const double *centroids,
                                           int32_t K, int32_t dim, float *database, int32_t *segment_counts) {
    return guard(__func__, [&]() -> int {
        if (segment_count < 0 || K < 0 || dim < 0 || (segment_count > 0 && !seg_cluster) ||
            (K > 0 && (!segment_counts || (dim > 0 && (!centroids || !database)))))
            return FA_STATUS_INVALID_ARGUMENT;
        reconstruct::build_speaker_database(seg_cluster, segment_count, centroids, K, dim, database, segment_counts);
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_speaker_constraints_resolve(int64_t num_embeddings, int64_t num_speakers, int64_t min_speakers,
                                                int64_t max_speakers, int64_t *resolved_min, int64_t *resolved_max) {
    return guard(__func__, [&]() -> int {
        if (!resolved_min || !resolved_max) return FA_STATUS_INVALID_ARGUMENT;
        long long lo = 0, hi = 0;
        kmeans::resolve_constraints(num_embeddings, num_speakers, min_speakers, max_speakers, &lo, &hi);
        *resolved_min = lo;
        *resolved_max = hi;
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_kmeans_cluster(const double *emb, size_t N, size_t D, int32_t num_clusters, int32_t max_iterations,
                                   int32_t n_init, uint64_t base_seed, int32_t *labels, double *centroids,
                                   int32_t centroid_cap, int32_t *centroid_rows, int32_t *best_init) {
    return guard(__func__, [&]() -> int {
        if (centroid_rows) *centroid_rows = 0;
        if (best_init) *best_init = 0;
        if (N == 0) return FA_STATUS_OK;                                  // :50-52
        if (!emb || !labels || max_iterations < 0) return FA_STATUS_INVALID_ARGUMENT;
        const long long rows_needed = D == 0 || num_clusters <= 0 ? 0 : std::min<long long>(num_clusters, (long long)N);
        if (rows_needed > 0 && (!centroids || centroid_cap < rows_needed)) return FA_STATUS_OUTPUT_TOO_SMALL;
        if (rows_needed == 0) {                                           // :53-58: dimension 0 or k <= 0 -> all zeros
            for (size_t i = 0; i < N; ++i) labels[i] = 0;
            return FA_STATUS_OK;
        }
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) {
            return kmeans_cluster(C, emb, N, D, num_clusters, max_iterations, n_init, base_seed, labels, centroids,
                                  centroid_rows, best_init);
        });
    });
}

FA_API fa_status fa_vbx_refine(const double *rho, size_t T, size_t D, const double *psi, size_t psi_len,
                               const int32_t *initial, int32_t S, const fa_vbx_config *cfg, double *gamma, double *pi,
                               double *elbos, int32_t *hard, int32_t *iterations) {
    return guard(__func__, [&]() -> int {
        if (!rho || !cfg || !gamma || !pi || !elbos || !hard || T == 0 || D == 0 || S <= 0)
            return FA_STATUS_INVALID_ARGUMENT;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) {
            return vbx_refine(C, rho, T, D, psi, psi_len, initial, S, *cfg, gamma, pi, elbos, hard, iterations);
        });
    });
}

FA_API fa_status fa_compute_centroids(const double *emb, size_t T, size_t dim, const double *gamma, const double *pi,
                                      int32_t S, double *centroids, int32_t *centroid_count) {
    return guard(__func__, [&]() -> int {
        if (!emb || !gamma || !pi || !centroids || !centroid_count || T == 0 || dim == 0 || S <= 0)
            return FA_STATUS_INVALID_ARGUMENT;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) {
            return compute_centroids(C, emb, T, dim, gamma, pi, S, centroids, centroid_count);
        });
    });
}

FA_API fa_status fa_assign_embeddings(const double *emb, size_t N, size_t dim, const double *centroids, int32_t K,
                                      int32_t *labels, double *scores) {
    return guard(__func__, [&]() -> int {
        if (N == 0) return FA_STATUS_OK;
        if (!emb || !labels || dim == 0 || (K > 0 && !centroids)) return FA_STATUS_INVALID_ARGUMENT;
        if (K <= 0) {   // guard !centroids.isEmpty else all zeros (:805-807)
            for (size_t i = 0; i < N; ++i) labels[i] = 0;
            return FA_STATUS_OK;
        }
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) {
            return assign_embeddings(C, emb, N, dim, centroids, K, labels, scores);
        });
    });
}

static int diarize_cluster(const float *emb256, const double *rho, size_t N, size_t emb_dim, size_t rho_dim,
                           const double *psi, const fa_cluster_config *cfg, const int32_t *chunk_index, int32_t *labels,
                           int32_t *initial, double *centroids, int32_t max_centroids, fa_cluster_info *info) {
    if (!emb256 || !rho || !cfg || !labels || N == 0 || emb_dim == 0 || rho_dim == 0) {
        fa::set_error("fa_diarize_cluster: null or empty input (the reference throws noSpeechDetected for N == 0)");
        return FA_STATUS_INVALID_ARGUMENT;
    }
    if (N > 0x7fffffffull / 4) return FA_STATUS_INDEX_OVERFLOW;
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) {
        return cluster_pipeline(C, emb256, rho, N, emb_dim, rho_dim, psi, *cfg, labels, initial, centroids, max_centroids,
                                info, chunk_index);
    });
}

FA_API fa_status fa_diarize_cluster(const float *emb256, const double *rho, size_t N, size_t emb_dim, size_t rho_dim,
                                    const double *psi, const fa_cluster_config *cfg, int32_t *labels, int32_t *initial,
                                    double *centroids, int32_t max_centroids, fa_cluster_info *info) {
    return guard(__func__, [&] {
        return diarize_cluster(emb256, rho, N, emb_dim, rho_dim, psi, cfg, nullptr, labels, initial, centroids,
                               max_centroids, info);
    });
}

FA_API fa_status fa_diarize_cluster_chunks(const float *emb256, const double *rho, size_t N, size_t emb_dim,
                                           size_t rho_dim, const double *psi, const fa_cluster_config *cfg,
                                           const int32_t *chunk_index, int32_t *labels, int32_t *initial,
                                           double *centroids, int32_t max_centroids, fa_cluster_info *info) {
    return guard(__func__, [&] {
        return diarize_cluster(emb256, rho, N, emb_dim, rho_dim, psi, cfg, chunk_index, labels, initial, centroids,
                               max_centroids, info);
    });
}

FA_API fa_status fa_hungarian_solve(const int64_t *cost, int32_t n, int32_t *assignment) {
    return guard(__func__, [&]() -> int {
        if (n < 0 || (n > 0 && (!cost || !assignment))) return FA_STATUS_INVALID_ARGUMENT;
        assign::min_cost_matching(cost, n, assignment);
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_max_score_assignment(const double *scores, int32_t rows, int32_t cols, int32_t *assignment) {
    return guard(__func__, [&]() -> int {
        if (rows < 0 || cols < 0 || (rows > 0 && !assignment) || (rows > 0 && cols > 0 && !scores))
            return FA_STATUS_INVALID_ARGUMENT;
        assign::max_score_matching(scores, rows, cols, assignment);
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_constrained_assign(const double *scores, size_t N, int32_t K, const int32_t *chunk_index,
                                       int32_t *labels) {
    return guard(__func__, [&]() -> int {
        if (N == 0) return FA_STATUS_OK;
        if (!chunk_index || !labels || K < 0 || (K > 0 && !scores)) return FA_STATUS_INVALID_ARGUMENT;
        assign::constrained_assign(scores, (long long)N, K, chunk_index, labels);
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_build_chunk_assignments(const int32_t *chunk_index, const int32_t *speaker_index,
                                            const int32_t *assignments, size_t N, int32_t num_chunks,
                                            int32_t num_speakers, int32_t cluster_count, int32_t *matrix) {
    return guard(__func__, [&]() -> int {
        if (num_chunks < 0 || num_speakers < 0 || (!matrix && (size_t)num_chunks * num_speakers > 0) ||
            (N > 0 && (!chunk_index || !speaker_index || !assignments)))
            return FA_STATUS_INVALID_ARGUMENT;
        assign::build_chunk_assignments(chunk_index, speaker_index, assignments, (long long)N, num_chunks, num_speakers,
                                        cluster_count, matrix);
        return FA_STATUS_OK;
    });
}

// The batch's argument checks; its lanes are cluster_batch (cluster_pipeline.cu).
static int cluster_batch_impl(const float *emb256, const double *rho, const int64_t *set_offsets, int32_t set_count,
                              size_t emb_dim, size_t rho_dim, const double *psi, const fa_cluster_config *cfg,
                              const int32_t *chunk_index, int32_t *labels, fa_cluster_info *infos) {
    if (!emb256 || !rho || !set_offsets || !cfg || !labels || set_count < 0 || emb_dim == 0 || rho_dim == 0)
        return FA_STATUS_INVALID_ARGUMENT;
    if (set_count == 0) return FA_STATUS_OK;
    if (set_offsets[0] < 0) {
        fa::set_error("fa_diarize_cluster_batch: set_offsets[0] = %lld is negative", (long long)set_offsets[0]);
        return FA_STATUS_INVALID_ARGUMENT;
    }
    for (int m = 0; m < set_count; ++m)
        if (set_offsets[m + 1] < set_offsets[m]) {
            fa::set_error("fa_diarize_cluster_batch: set_offsets decrease at set %d (%lld -> %lld)", m,
                          (long long)set_offsets[m], (long long)set_offsets[m + 1]);
            return FA_STATUS_INVALID_ARGUMENT;
        }
    if (infos)   // an empty set is not clustered: its info reads all zeros
        for (int m = 0; m < set_count; ++m)
            if (set_offsets[m + 1] == set_offsets[m]) infos[m] = fa_cluster_info{};
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return cluster_batch(emb256, rho, set_offsets, set_count, emb_dim, rho_dim, psi, *cfg, chunk_index, labels, infos);
}

FA_API fa_status fa_diarize_cluster_batch(const float *emb256, const double *rho, const int64_t *set_offsets,
                                          int32_t set_count, size_t emb_dim, size_t rho_dim, const double *psi,
                                          const fa_cluster_config *cfg, int32_t *labels, fa_cluster_info *infos) {
    return guard(__func__, [&] {
        return cluster_batch_impl(emb256, rho, set_offsets, set_count, emb_dim, rho_dim, psi, cfg, nullptr, labels,
                                  infos);
    });
}

// The reference's default (constrained) assignment per set: chunk_index[row] = TimedEmbedding.chunkIndex of that row,
// numbered inside its own set.
FA_API fa_status fa_diarize_cluster_batch_chunks(const float *emb256, const double *rho, const int64_t *set_offsets,
                                                 int32_t set_count, size_t emb_dim, size_t rho_dim, const double *psi,
                                                 const fa_cluster_config *cfg, const int32_t *chunk_index,
                                                 int32_t *labels, fa_cluster_info *infos) {
    return guard(__func__, [&] {
        return cluster_batch_impl(emb256, rho, set_offsets, set_count, emb_dim, rho_dim, psi, cfg, chunk_index, labels,
                                  infos);
    });
}

// ------------------------------------------------------------------------------------------------ prepare stage
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
    if ((long long)first_chunk + chunk_count > prepare::window_count(total_samples, c)) {
        fa::set_error("fa_seg_windows: chunks %d .. %lld lie past the last window", first_chunk,
                      (long long)first_chunk + chunk_count - 1);
        return FA_STATUS_INVALID_ARGUMENT;
    }
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
        !(plan_cfg->min_segment_duration >= 0.0)) {
        fa::set_error("fa_embed_plan_config: weight_frames, audio_sample_count and fbank_batch must be positive and "
                      "min_segment_duration >= 0");
        return FA_STATUS_INVALID_ARGUMENT;
    }
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

// ------------------------------------------------------------------------------------------------ Sortformer state
// SortformerStateUpdater.streamingUpdate for many sessions in HBM: sortformer_streams.cu, sortformer_kernels.cu.
static sortformer::Config sortformer_config_of(const fa_sortformer_config *c) {
    sortformer::Config s{};
    s.chunk_len = c->chunk_len;
    s.left_context = c->chunk_left_context;
    s.right_context = c->chunk_right_context;
    s.fifo_len = c->fifo_len;
    s.spkcache_len = c->spkcache_len;
    s.update_period = c->spkcache_update_period;
    s.sil_per_spk = c->spkcache_sil_frames_per_spk;
    s.silence_threshold = c->silence_threshold;
    s.pred_score_threshold = c->pred_score_threshold;
    s.scores_boost_latest = c->scores_boost_latest;
    s.strong_boost_rate = c->strong_boost_rate;
    s.weak_boost_rate = c->weak_boost_rate;
    s.min_pos_scores_rate = c->min_pos_scores_rate;
    return s;
}

FA_API fa_status fa_sortformer_default_config(fa_sortformer_config *cfg, int32_t preset) {
    return guard(__func__, [&]() -> int {
        if (!cfg) return FA_STATUS_INVALID_ARGUMENT;
        // SortformerTypes.swift:121-216: chunkLen, left, right context, fifoLen, spkcacheLen, update period
        static const int32_t presets[8][6] = {
            {6, 1, 7, 40, 188, 31},    {6, 1, 7, 40, 188, 31},   {6, 1, 7, 40, 188, 31},   {6, 1, 7, 188, 188, 144},
            {6, 1, 7, 188, 188, 144},  {340, 1, 40, 40, 188, 300}, {340, 1, 40, 40, 188, 300}, {25, 1, 7, 40, 188, 31},
        };
        if (preset < 0 || preset > 7) {
            fa::set_error("fa_sortformer_default_config: unknown preset %d", preset);
            return FA_STATUS_INVALID_ARGUMENT;
        }
        const int32_t *p = presets[preset];
        // the init's defaults (SortformerTypes.swift:219-236) and its clamps, as the static configs hold them:
        // highContext's period 300 becomes chunkLen = 340
        *cfg = fa_sortformer_config{p[0], p[1], p[2], p[3], p[4], p[5], 3, 0.2f, 0.25f, 0.05f, 0.75f, 1.5f, 0.5f};
        cfg->spkcache_update_period = std::max(std::min(p[5], p[3] + p[0]), p[0]);
        return FA_STATUS_OK;
    });
}

static void sortformer_config_out(const sortformer::Config &c, fa_sortformer_config *o) {
    *o = fa_sortformer_config{c.chunk_len, c.left_context, c.right_context, c.fifo_len, c.spkcache_len, c.update_period,
                              c.sil_per_spk, c.silence_threshold, c.pred_score_threshold, c.scores_boost_latest,
                              c.strong_boost_rate, c.weak_boost_rate, c.min_pos_scores_rate};
}

FA_API fa_status fa_sortformer_resolve_config(const fa_sortformer_config *cfg, int32_t max_core_frames,
                                              fa_sortformer_config *resolved, int32_t *resolved_max_core) {
    return guard(__func__, [&]() -> int {
        if (!cfg) return FA_STATUS_INVALID_ARGUMENT;
        sortformer::Config c;
        const int st = sortformer::resolve_config(sortformer_config_of(cfg), max_core_frames, c);
        if (st != FA_OK) return st;
        if (resolved) sortformer_config_out(c, resolved);
        if (resolved_max_core) *resolved_max_core = c.max_core;
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_sortformer_step(const fa_sortformer_config *cfg, int32_t max_core_frames, const int32_t *lengths_in,
                                    int32_t emb_length, int32_t pred_rows, int32_t left_context, int32_t right_context,
                                    int32_t *out) {
    return guard(__func__, [&]() -> int {
        if (!cfg || !lengths_in || !out) return FA_STATUS_INVALID_ARGUMENT;
        sortformer::Config c;
        int st = sortformer::resolve_config(sortformer_config_of(cfg), max_core_frames, c);
        if (st != FA_OK) return st;
        if (lengths_in[0] < 0 || lengths_in[0] > c.spkcache_len || lengths_in[1] < 0 || lengths_in[1] > c.fifo_len) {
            fa::set_error("fa_sortformer_step: lengths (%d, %d) outside the state's bounds", lengths_in[0], lengths_in[1]);
            return FA_STATUS_INVALID_ARGUMENT;
        }
        sortformer::Step s;
        st = sortformer::plan_step(c, lengths_in[0], lengths_in[1], lengths_in[2] != 0, emb_length, pred_rows,
                                   left_context, right_context, s);
        if (st != FA_OK) return st;
        const int32_t v[6] = {s.core, s.pop, s.compress, s.spkcache_after, s.fifo_after, s.has_preds_after};
        std::memcpy(out, v, sizeof(v));
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_sortformer_create(const fa_sortformer_config *cfg, int32_t max_core_frames, fa_sortformer **out) {
    return guard(__func__, [&]() -> int {
        if (!cfg || !out) return FA_STATUS_INVALID_ARGUMENT;
        *out = nullptr;
        sortformer::Config c;
        int st = sortformer::resolve_config(sortformer_config_of(cfg), max_core_frames, c);
        if (st != FA_OK) return st;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        std::unique_ptr<fa_sortformer> h(new fa_sortformer());
        st = h->set.init(c);
        if (st != FA_OK) return st;
        *out = h.release();
        return FA_STATUS_OK;
    });
}

FA_API void fa_sortformer_destroy(fa_sortformer *h) { delete h; }

FA_API fa_status fa_sortformer_open(fa_sortformer *h, int32_t *session) {
    return guard(__func__, [&]() -> int {
        if (!h || !session) return FA_STATUS_INVALID_ARGUMENT;
        int id = -1;
        const int st = h->set.open(&id);
        if (st == FA_OK) *session = id;
        return st;
    });
}

FA_API fa_status fa_sortformer_close(fa_sortformer *h, int32_t session) {
    return guard(__func__, [&]() -> int {
        if (!h) return FA_STATUS_INVALID_ARGUMENT;
        return h->set.close(session);
    });
}

static int sortformer_update(fa_sortformer *h, int32_t count, const int32_t *sessions, const float *embs,
                             int32_t emb_rows, const float *preds, int32_t pred_rows, const int32_t *emb_lengths,
                             const int32_t *left, const int32_t *right, bool device, float *confirmed,
                             size_t confirmed_len, float *tentative, size_t tentative_len, int64_t *confirmed_rows,
                             int64_t *tentative_rows) {
    if (!h) return FA_STATUS_INVALID_ARGUMENT;
    return h->set.update(count, sessions, embs, emb_rows, preds, pred_rows, emb_lengths, left, right, device, confirmed,
                         capacity(confirmed_len), tentative, capacity(tentative_len), confirmed_rows, tentative_rows);
}

FA_API fa_status fa_sortformer_update(fa_sortformer *h, int32_t count, const int32_t *sessions, const float *chunk_embs,
                                      int32_t emb_rows, const float *preds, int32_t pred_rows, const int32_t *emb_lengths,
                                      const int32_t *left_context, const int32_t *right_context, float *confirmed,
                                      size_t confirmed_len, float *tentative, size_t tentative_len,
                                      int64_t *confirmed_rows, int64_t *tentative_rows) {
    return guard(__func__, [&] {
        return sortformer_update(h, count, sessions, chunk_embs, emb_rows, preds, pred_rows, emb_lengths, left_context,
                                 right_context, false, confirmed, confirmed_len, tentative, tentative_len,
                                 confirmed_rows, tentative_rows);
    });
}

FA_API fa_status fa_sortformer_update_device(fa_sortformer *h, int32_t count, const int32_t *sessions,
                                             const float *d_chunk_embs, int32_t emb_rows, const float *d_preds,
                                             int32_t pred_rows, const int32_t *emb_lengths, const int32_t *left_context,
                                             const int32_t *right_context, float *d_confirmed, size_t confirmed_len,
                                             float *d_tentative, size_t tentative_len, int64_t *confirmed_rows,
                                             int64_t *tentative_rows) {
    return guard(__func__, [&] {
        return sortformer_update(h, count, sessions, d_chunk_embs, emb_rows, d_preds, pred_rows, emb_lengths,
                                 left_context, right_context, true, d_confirmed, confirmed_len, d_tentative,
                                 tentative_len, confirmed_rows, tentative_rows);
    });
}

static int sortformer_inputs(fa_sortformer *h, int32_t count, const int32_t *sessions, bool device, float *spkcache,
                             float *fifo, int32_t *spkcache_lengths, int32_t *fifo_lengths) {
    if (!h) return FA_STATUS_INVALID_ARGUMENT;
    return h->set.model_inputs(count, sessions, device, spkcache, fifo, spkcache_lengths, fifo_lengths);
}

FA_API fa_status fa_sortformer_model_inputs(fa_sortformer *h, int32_t count, const int32_t *sessions, float *spkcache,
                                            float *fifo, int32_t *spkcache_lengths, int32_t *fifo_lengths) {
    return guard(__func__, [&] {
        return sortformer_inputs(h, count, sessions, false, spkcache, fifo, spkcache_lengths, fifo_lengths);
    });
}

FA_API fa_status fa_sortformer_model_inputs_device(fa_sortformer *h, int32_t count, const int32_t *sessions,
                                                   float *d_spkcache, float *d_fifo, int32_t *spkcache_lengths,
                                                   int32_t *fifo_lengths) {
    return guard(__func__, [&] {
        return sortformer_inputs(h, count, sessions, true, d_spkcache, d_fifo, spkcache_lengths, fifo_lengths);
    });
}

FA_API fa_status fa_sortformer_session_state(fa_sortformer *h, int32_t session, fa_sortformer_session_info *info,
                                             float *spkcache, float *spkcache_preds, float *fifo, float *fifo_preds,
                                             float *mean_silence) {
    return guard(__func__, [&]() -> int {
        if (!h || !info) return FA_STATUS_INVALID_ARGUMENT;
        sortformer::SessionInfo s;
        const int st = h->set.state(session, &s, spkcache, spkcache_preds, fifo, fifo_preds, mean_silence);
        if (st != FA_OK) return st;
        *info = fa_sortformer_session_info{s.spkcache_length, s.fifo_length, s.has_spkcache_preds, s.has_fifo_preds,
                                           s.chunks,          s.silence_frames};
        return FA_STATUS_OK;
    });
}

// ------------------------------------------------------------------------------------------------ diarizer timelines
// DiarizerTimeline's numeric core for many sessions in HBM: timeline_streams.cu, timeline_kernels.cu.
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
            fa::set_error("fa_diarizer_timeline_default_config: unknown preset %d", preset);
            return FA_STATUS_INVALID_ARGUMENT;
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
            if (!(r >= -2147483648.0f && r < 2147483648.0f)) {
                fa::set_error("fa_diarizer_timeline_config_from_seconds: %g s / %g s is not a finite int32 frame count",
                              (double)secs[k], (double)cfg->frame_duration_seconds);
                return FA_STATUS_INVALID_ARGUMENT;
            }
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
