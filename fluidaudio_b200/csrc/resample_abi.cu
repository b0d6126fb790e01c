// C ABI of the converter stage (declared in include/fluidaudio_b200.h) over resample_kernels.cu.  Every entry point
// that returns a status returns through guard() (c_abi.h).
#include "c_abi.h"
#include "resample_plan.h"

namespace fa {
namespace resample {

bool audio_format_ok(const fa_audio_format *f) {
    if (!f || !(f->in_rate > 0) || !(f->out_rate > 0) || f->channels < 1 || f->channels > 64 ||
        (f->format != FA_PCM_F32 && f->format != FA_PCM_I16) || f->algorithm < 0 || f->algorithm > 2) {
        fa::set_error("audio format: rates must be positive, 1..64 channels, format F32/I16, algorithm 0..2");
        return false;
    }
    return true;
}
AudioFormat to_format(const fa_audio_format *f) {
    return AudioFormat{f->in_rate, f->out_rate, f->channels, f->format, f->interleaved ? 1 : 0, f->algorithm};
}

} // namespace resample
} // namespace fa

using namespace fa;

FA_API int64_t fa_resample_output_count(const fa_audio_format *fmt, int64_t frames) {
    if (!fmt || frames < 0 || !(fmt->in_rate > 0) || !(fmt->out_rate > 0)) {
        fa::set_error("fa_resample_output_count: fmt is NULL, frames < 0 or a rate is not positive");
        return -1;
    }
    return resample::output_count(frames, fmt->in_rate, fmt->out_rate);
}

static int audio_resample(const void *pcm, int64_t frames, const fa_audio_format *fmt, float *out, int64_t out_cap,
                          int64_t *out_count) {
    if (!resample::audio_format_ok(fmt) || frames < 0 || !out_count) return FA_STATUS_INVALID_ARGUMENT;
    const long long n = resample::output_count(frames, fmt->in_rate, fmt->out_rate);
    *out_count = n;
    if (!out) return FA_STATUS_OK;            // sizing call: pcm may be NULL
    if (!pcm && frames) return refuse("fa_audio_resample: pcm is NULL");
    if (out_cap < n) return FA_STATUS_OUTPUT_TOO_SMALL;
    if (n == 0) return FA_STATUS_OK;
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return resample::convert_host(pcm, frames, resample::to_format(fmt), out, n);
}

FA_API fa_status fa_audio_resample(const void *pcm, int64_t frames, const fa_audio_format *fmt, float *out,
                                   int64_t out_cap, int64_t *out_count) {
    return guard(__func__, [&] { return audio_resample(pcm, frames, fmt, out, out_cap, out_count); });
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
