// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
//
// CPU restatement (plain C++, single thread, pinned FP flags: no contraction) of the reference's three torch-style
// log-mel frontends, line by line:
//   Cohere     Sources/FluidAudio/ASR/Cohere/CoherePipeline.swift:41-324  CohereMelSpectrogram (init :86-118, compute
//              :127-247, padOrTruncate :250-263, slaneyMelFilter :273-323)
//   StyleTTS2  Sources/FluidAudio/TTS/StyleTTS2/Pipeline/Preprocess/StyleTTS2MelExtractor.swift (compute :77-141,
//              hannWindowPadded :148-158, htkMelFilterbank :160-221, reflectPad :226-250)
//   LuxTTS     Sources/FluidAudio/TTS/LuxTts/LuxTtsMelExtractor.swift (extract :52-132, tables :152-187)
// Everything is float32 in the order the Swift states it (LuxTTS's table float64), with two conventions:
//   * the DFT (vDSP, closed) is the float32 frame's DFT evaluated in float64 and rounded ONCE to float32, the
//     implementation-independent value oracle_mel.cpp uses (vDSP's packed real FFT returns 2X; the Swift's * 0.5 undoes it
//     exactly, so X is used directly);
//   * the vDSP mat-vec / dot products are sequential float32 sums in bin order, and vDSP_vthr is Swift's max (a NaN mel
//     stays NaN).
// Cohere's pre-emphasis keeps the Swift's two roundings: x[i] - (a * x[i-1]).
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

float swift_float_pi() {   // Swift's Float.pi is pi rounded toward zero
    const uint32_t bits = 0x40490FDAu;
    float f;
    std::memcpy(&f, &bits, 4);
    return f;
}
template <typename T> T smin(T x, T y) { return y < x ? y : x; }   // Swift.min
template <typename T> T smax(T x, T y) { return y >= x ? y : x; }  // Swift.max

// DFT of a real float32 frame, float64 radix-2, bins 0..n/2 rounded once to float32
struct Dft {
    int n = 0, lg = 0;
    std::vector<double> cs, sn, re, im;
    std::vector<int> rev;
    explicit Dft(int n_) : n(n_), cs(n_), sn(n_), re(n_), im(n_), rev(n_) {
        while ((1 << lg) < n) ++lg;
        for (int k = 0; k < n; ++k) {
            const double a = 2.0 * M_PI * (double)k / (double)n;
            cs[k] = std::cos(a);
            sn[k] = std::sin(a);
        }
        for (int i = 0; i < n; ++i) {
            int r = 0;
            for (int b = 0; b < lg; ++b)
                if (i & (1 << b)) r |= 1 << (lg - 1 - b);
            rev[i] = r;
        }
    }
    void run(const float *frame, float *out_re, float *out_im) {
        for (int i = 0; i < n; ++i) {
            re[rev[i]] = (double)frame[i];
            im[rev[i]] = 0.0;
        }
        for (int len = 2; len <= n; len <<= 1) {
            const int half = len >> 1, step = n / len;
            for (int base = 0; base < n; base += len)
                for (int j = 0; j < half; ++j) {
                    const double wr = cs[j * step], wi = -sn[j * step];
                    const int a = base + j, b = a + half;
                    const double tr = re[b] * wr - im[b] * wi, ti = re[b] * wi + im[b] * wr;
                    re[b] = re[a] - tr;
                    im[b] = im[a] - ti;
                    re[a] = re[a] + tr;
                    im[a] = im[a] + ti;
                }
        }
        for (int b = 0; b <= n / 2; ++b) {
            out_re[b] = (float)re[b];
            out_im[b] = (float)im[b];
        }
    }
};

int next_pow2(int n) {
    int x = 1;
    while (x < n) x <<= 1;
    return x;
}

float cohere_hz_to_mel(float hz) {
    const float f_sp = 200.0f / 3.0f;
    if (hz >= 1000.0f) return 15.0f + logf(hz / 1000.0f) / 0.06875177742f;
    return hz / f_sp;
}
float cohere_mel_to_hz(float mel) {
    const float f_sp = 200.0f / 3.0f;
    if (mel >= 15.0f) return 1000.0f * expf(0.06875177742f * (mel - 15.0f));
    return f_sp * mel;
}

}  // namespace

extern "C" {

// ---------------------------------------------------------------------------------------------------------- Cohere
// window: the winLength symmetric Hann (:90-97; a length-1 window is [0])
void oracle_cohere_window(int32_t win_length, float *out) {
    for (int n = 0; n < win_length; ++n) out[n] = 0.0f;
    if (win_length > 1) {
        const float denom = (float)(win_length - 1), pi = swift_float_pi();
        for (int n = 0; n < win_length; ++n) out[n] = 0.5f * (1.0f - cosf(2.0f * pi * (float)n / denom));
    }
}

// [n_mels x (n_fft/2+1)] (:273-303)
void oracle_cohere_filterbank(int32_t sample_rate, int32_t n_fft, int32_t n_mels, float f_min, float f_max, float *out) {
    const int bins = n_fft / 2 + 1;
    std::vector<float> freqs(bins), pts(n_mels + 2), hz(n_mels + 2);
    for (int k = 0; k < bins; ++k) freqs[k] = (float)sample_rate * (float)k / (float)n_fft;
    const float mel_min = cohere_hz_to_mel(f_min), mel_max = cohere_hz_to_mel(f_max);
    const float step = (mel_max - mel_min) / (float)(n_mels + 1);
    for (int i = 0; i < n_mels + 2; ++i) pts[i] = mel_min + (float)i * step;
    for (int i = 0; i < n_mels + 2; ++i) hz[i] = cohere_mel_to_hz(pts[i]);
    for (int64_t i = 0; i < (int64_t)n_mels * bins; ++i) out[i] = 0.0f;
    for (int m = 0; m < n_mels; ++m) {
        const float lower = hz[m], center = hz[m + 1], upper = hz[m + 2];
        const float left_den = smax(center - lower, 1e-10f), right_den = smax(upper - center, 1e-10f);
        float *row = out + (int64_t)m * bins;
        for (int k = 0; k < bins; ++k) {
            const float f = freqs[k];
            if (f < lower || f > upper) continue;
            row[k] = (f <= center) ? (f - lower) / left_den : (upper - f) / right_den;
        }
        const float enorm = 2.0f / smax(upper - lower, 1e-10f);
        for (int k = 0; k < bins; ++k) row[k] *= enorm;
    }
}

// CohereMelSpectrogram.compute (:127-247).  out: [n_mels x T], T = 1 + n / hop (returned); *valid = n / hop.
int64_t oracle_cohere_compute(int32_t sample_rate, int32_t win_length, int32_t hop, int32_t n_mels, float f_min,
                              float f_max, float preemph, float mag_power, float log_guard, float cmvn_eps,
                              const float *audio, int64_t count, float *out, int64_t *valid_out) {
    const int n_fft = next_pow2(win_length), bins = n_fft / 2 + 1, pad = n_fft / 2;
    const int64_t valid = (count > 0 ? count : 0) / hop;
    std::vector<float> samples(audio, audio + count);
    if (preemph != 0.0f && count > 1) {
        std::vector<float> filtered(count, 0.0f);
        filtered[0] = samples[0];
        for (int64_t i = 1; i < count; ++i) {
            const float t = preemph * samples[i - 1];
            filtered[i] = samples[i] - t;
        }
        samples.swap(filtered);
    }
    std::vector<float> padded(count + 2 * pad, 0.0f);
    for (int64_t i = 0; i < count; ++i) padded[pad + i] = samples[i];
    const int64_t frames = 1 + ((int64_t)padded.size() - n_fft) / hop;
    std::vector<float> hann(win_length), window(n_fft, 0.0f), fb((size_t)n_mels * bins);
    oracle_cohere_window(win_length, hann.data());
    if (win_length < n_fft) {
        const int left = (n_fft - win_length) / 2;
        for (int i = 0; i < win_length; ++i) window[left + i] = hann[i];
    } else {
        window = hann;
    }
    oracle_cohere_filterbank(sample_rate, n_fft, n_mels, f_min, f_max, fb.data());
    Dft dft(n_fft);
    std::vector<float> frame(n_fft), re(bins), im(bins), power((size_t)bins * frames);
    for (int64_t f = 0; f < frames; ++f) {
        for (int i = 0; i < n_fft; ++i) frame[i] = padded[f * hop + i] * window[i];
        dft.run(frame.data(), re.data(), im.data());
        for (int k = 0; k < bins; ++k) {
            const float a = re[k] * re[k], b = im[k] * im[k];
            const float mag = sqrtf(a + b);   // DC / Nyquist: abs(real) = sqrt(real^2) exactly
            power[(size_t)k * frames + f] = powf(mag, mag_power);
        }
    }
    for (int m = 0; m < n_mels; ++m) {
        const float *filt = &fb[(size_t)m * bins];
        for (int64_t f = 0; f < frames; ++f) {
            float sum = 0.0f;
            for (int k = 0; k < bins; ++k) {
                const float t = filt[k] * power[(size_t)k * frames + f];
                sum += t;
            }
            out[m * frames + f] = logf(sum + log_guard);
        }
    }
    if (valid > 1) {
        for (int m = 0; m < n_mels; ++m) {
            float *row = out + m * frames;
            float mean = 0.0f;
            for (int64_t f = 0; f < valid; ++f) mean += row[f];
            mean /= (float)valid;
            float ssq = 0.0f;
            for (int64_t f = 0; f < valid; ++f) {
                const float d = row[f] - mean;
                const float dd = d * d;
                ssq += dd;
            }
            const float variance = ssq / (float)(valid - 1);
            float sd = sqrtf(variance);
            if (!std::isfinite(sd)) sd = 0.0f;
            const float denom = sd + cmvn_eps;
            for (int64_t f = 0; f < valid; ++f) row[f] = (row[f] - mean) / denom;
        }
    }
    for (int m = 0; m < n_mels; ++m)
        for (int64_t f = valid; f < frames; ++f) out[m * frames + f] = 0.0f;
    *valid_out = valid;
    return frames;
}

// Cohere's CMVN, invalid-frame zeroing and padOrTruncate applied to a given log-mel: x [T x n_mels] time-major (the
// library's own log-mel), out [n_mels x fixed] (fixed < 0: T).  Returns the output width.
int64_t oracle_cohere_cmvn(const float *x, int64_t T, int32_t n_mels, int64_t valid, int64_t fixed, float cmvn_eps,
                           float *out) {
    const int64_t W = fixed < 0 ? T : fixed;
    std::vector<float> row(T);
    for (int m = 0; m < n_mels; ++m) {
        for (int64_t t = 0; t < T; ++t) row[t] = x[t * n_mels + m];
        if (valid > 1) {
            float mean = 0.0f;
            for (int64_t f = 0; f < valid; ++f) mean += row[f];
            mean /= (float)valid;
            float ssq = 0.0f;
            for (int64_t f = 0; f < valid; ++f) {
                const float d = row[f] - mean;
                const float dd = d * d;
                ssq += dd;
            }
            float sd = sqrtf(ssq / (float)(valid - 1));
            if (!std::isfinite(sd)) sd = 0.0f;
            const float denom = sd + cmvn_eps;
            for (int64_t f = 0; f < valid; ++f) row[f] = (row[f] - mean) / denom;
        }
        for (int64_t f = valid; f < T; ++f) row[f] = 0.0f;
        for (int64_t t = 0; t < W; ++t) out[m * W + t] = t < T ? row[t] : 0.0f;
    }
    return W;
}

// ------------------------------------------------------------------------------------------------------ reflect pad
// StyleTTS2MelExtractor.reflectPad (:226-250): out has n + 2 pad samples (2 pad zeros for an empty clip).
void oracle_reflect_pad(const float *x, int64_t n, int32_t pad, float *out) {
    if (n == 0) {
        for (int i = 0; i < 2 * pad; ++i) out[i] = 0.0f;
        return;
    }
    for (int i = 0; i < pad; ++i) out[i] = x[smin<int64_t>(pad - i, n - 1)];
    for (int64_t i = 0; i < n; ++i) out[pad + i] = x[i];
    for (int i = 0; i < pad; ++i) out[pad + n + i] = x[smax<int64_t>(n - 2 - i, 0)];
}

// -------------------------------------------------------------------------------------------------------- StyleTTS2
// periodic Hann centred in n_fft (:148-158)
void oracle_styletts2_window(int32_t win_length, int32_t n_fft, float *out) {
    for (int i = 0; i < n_fft; ++i) out[i] = 0.0f;
    const float two_pi = swift_float_pi() * 2.0f, denom = (float)win_length;
    const int pad = (n_fft - win_length) / 2;
    for (int n = 0; n < win_length; ++n) out[pad + n] = 0.5f * (1.0f - cosf(two_pi * (float)n / denom));
}

// htkMelFilterbank (:174-221), fMin 0, fMax sample_rate / 2
void oracle_styletts2_filterbank(int32_t n_mels, int32_t n_fft, int32_t sample_rate, float *out) {
    const int bins = n_fft / 2 + 1;
    auto to_mel = [](float hz) { return 2595.0f * log10f(1.0f + hz / 700.0f); };
    auto to_hz = [](float mel) { return 700.0f * (powf(10.0f, mel / 2595.0f) - 1.0f); };
    std::vector<float> freqs(bins), hz(n_mels + 2);
    const float bin_step = (float)sample_rate / (float)n_fft;
    for (int k = 0; k < bins; ++k) freqs[k] = (float)k * bin_step;
    const float mel_min = to_mel(0.0f), mel_max = to_mel((float)sample_rate / 2.0f);
    for (int i = 0; i < n_mels + 2; ++i) {
        const float frac = (float)i / (float)(n_mels + 1);
        hz[i] = to_hz(mel_min + (mel_max - mel_min) * frac);
    }
    for (int64_t i = 0; i < (int64_t)n_mels * bins; ++i) out[i] = 0.0f;
    for (int m = 0; m < n_mels; ++m) {
        const float left = hz[m], center = hz[m + 1], right = hz[m + 2];
        const float left_slope = center - left, right_slope = right - center;
        for (int k = 0; k < bins; ++k) {
            const float f = freqs[k];
            if (f < left || f > right) continue;
            float val;
            if (f <= center) val = left_slope > 0 ? (f - left) / left_slope : 0.0f;
            else val = right_slope > 0 ? (right - f) / right_slope : 0.0f;
            out[(int64_t)m * bins + k] = smax(val, 0.0f);
        }
    }
}

// compute (:77-141): out [n_mels x frames], frames = 1 + n / hop returned.  affine = 0 leaves log(mel + eps) as it is.
int64_t oracle_styletts2_compute(int32_t n_fft, int32_t win_length, int32_t hop, int32_t n_mels, int32_t filter_sr,
                                 float mean, float std_, float log_eps, int32_t affine, const float *audio, int64_t n,
                                 float *out) {
    const int pad = n_fft / 2, bins = n_fft / 2 + 1;
    std::vector<float> padded(n + 2 * pad), window(n_fft), fb((size_t)n_mels * bins);
    oracle_reflect_pad(audio, n, pad, padded.data());
    const int64_t usable = (int64_t)padded.size() - n_fft;
    const int64_t frames = usable >= 0 ? usable / hop + 1 : 0;
    oracle_styletts2_window(win_length, n_fft, window.data());
    oracle_styletts2_filterbank(n_mels, n_fft, filter_sr, fb.data());
    Dft dft(n_fft);
    std::vector<float> frame(n_fft), re(bins), im(bins), power(bins);
    for (int64_t f = 0; f < frames; ++f) {
        for (int i = 0; i < n_fft; ++i) frame[i] = padded[f * hop + i] * window[i];
        dft.run(frame.data(), re.data(), im.data());
        for (int k = 0; k < bins; ++k) {
            const float a = re[k] * re[k], b = im[k] * im[k];
            power[k] = a + b;
        }
        for (int m = 0; m < n_mels; ++m) {
            float acc = 0.0f;
            for (int k = 0; k < bins; ++k) {
                const float t = fb[(size_t)m * bins + k] * power[k];
                acc += t;
            }
            const float l = logf(acc + log_eps);
            out[m * frames + f] = affine ? (l - mean) / std_ : l;
        }
    }
    return frames;
}

// ------------------------------------------------------------------------------------------------------------ LuxTTS
void oracle_luxtts_window(int32_t length, float *out) {   // periodicHannWindow (:152-156)
    const float pi = swift_float_pi();
    for (int i = 0; i < length; ++i) out[i] = 0.5f * (1.0f - cosf(2.0f * pi * (float)i / (float)length));
}

// htkMelFilterbank (:160-187), Double
void oracle_luxtts_filterbank(int32_t n_fft, int32_t n_mels, int32_t sample_rate, float *out) {
    const int bins = n_fft / 2 + 1;
    const double f_max = (double)sample_rate / 2.0;
    auto to_mel = [](double hz) { return 2595.0 * log10(1.0 + hz / 700.0); };
    auto to_hz = [](double mel) { return 700.0 * (pow(10.0, mel / 2595.0) - 1.0); };
    const double mel_min = to_mel(0.0), mel_max = to_mel(f_max);
    std::vector<double> pts(n_mels + 2), freqs(bins);
    for (int i = 0; i < n_mels + 2; ++i) pts[i] = to_hz(mel_min + (double)i * (mel_max - mel_min) / (double)(n_mels + 1));
    for (int b = 0; b < bins; ++b) freqs[b] = (double)b * f_max / (double)(bins - 1);
    for (int m = 0; m < n_mels; ++m)
        for (int b = 0; b < bins; ++b) {
            const double up = (freqs[b] - pts[m]) / (pts[m + 1] - pts[m]);
            const double down = (pts[m + 2] - freqs[b]) / (pts[m + 2] - pts[m + 1]);
            out[(int64_t)m * bins + b] = (float)smax(0.0, smin(up, down));
        }
}

// extract (:52-132): out [T x n_mels], T = (n + hop/2) / hop returned (0 for n == 0).  Frames past the STFT's count
// replicate the last one (:126-130).
int64_t oracle_luxtts_extract(int32_t n_fft, int32_t hop, int32_t n_mels, int32_t sample_rate, float log_floor,
                              const float *audio, int64_t n, float *out) {
    const int64_t target = (n + hop / 2) / hop;
    if (n <= 0 || target <= 0) return 0;
    const int pad = n_fft / 2, bins = n_fft / 2 + 1;
    std::vector<float> padded(n + 2 * pad, 0.0f), window(n_fft), fb((size_t)n_mels * bins);
    for (int i = 0; i < pad; ++i) {
        padded[i] = audio[smin<int64_t>(pad - i, n - 1)];
        padded[pad + n + i] = audio[smax<int64_t>(n - 2 - i, 0)];
    }
    for (int64_t i = 0; i < n; ++i) padded[pad + i] = audio[i];
    const int64_t stft = 1 + n / hop;
    oracle_luxtts_window(n_fft, window.data());
    oracle_luxtts_filterbank(n_fft, n_mels, sample_rate, fb.data());
    Dft dft(n_fft);
    std::vector<float> frame(n_fft), re(bins), im(bins), mag(bins);
    int64_t made = 0;
    for (int64_t f = 0; f < smin(stft, target); ++f, ++made) {
        for (int i = 0; i < n_fft; ++i) frame[i] = padded[f * hop + i] * window[i];
        dft.run(frame.data(), re.data(), im.data());
        for (int k = 0; k < bins; ++k) {
            const float a = re[k] * re[k], b = im[k] * im[k];
            mag[k] = sqrtf(a + b);
        }
        for (int m = 0; m < n_mels; ++m) {
            float acc = 0.0f;
            for (int k = 0; k < bins; ++k) {
                const float t = fb[(size_t)m * bins + k] * mag[k];
                acc += t;
            }
            out[f * n_mels + m] = logf(smax(acc, log_floor));
        }
    }
    for (; made < target; ++made)
        for (int m = 0; m < n_mels; ++m) out[made * n_mels + m] = out[(made - 1) * n_mels + m];
    return target;
}

}  // extern "C"
