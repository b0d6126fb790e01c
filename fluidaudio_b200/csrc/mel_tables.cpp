// Host tables of the log-mel plan (mel_tables.h): the window and filterbank builders of every reference class, the ex
// config check, and the packed filterbank format the kernels read (bands, mel512_kernel's schedule, weights, window
// placements).
#include "mel_tables.h"
#include "mel_core.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace fa {
namespace mel {

static float swift_float_pi() {
    const uint32_t bits = 0x40490FDAu;   // Swift's Float.pi is rounded toward zero
    float f;
    std::memcpy(&f, &bits, 4);
    return f;
}

// AudioMelSpectrogram.swift:553-562
static void build_window(int length, bool periodic, std::vector<float> &w) {
    w.resize(length);
    const float divisor = periodic ? (float)length : (float)(length - 1);
    const float pi = swift_float_pi();
    for (int i = 0; i < length; ++i) {
        const float phase = 2.0f * pi * (float)i / divisor;
        w[i] = 0.5f * (1.0f - cosf(phase));
    }
}

// AudioMelSpectrogram.swift:564-642 (Slaney mel scale, Slaney area normalisation, Float32 arithmetic)
static void build_filterbank(int n_fft, int n_mels, int sample_rate, std::vector<float> &fb) {
    const int bins = n_fft / 2 + 1;
    const float f_sp = 200.0f / 3.0f, min_log_hz = 1000.0f;
    const float min_log_mel = min_log_hz / f_sp;
    const float log_step = logf(6.4f) / 27.0f;
    auto to_mel = [&](float hz) { return hz >= min_log_hz ? min_log_mel + logf(hz / min_log_hz) / log_step : hz / f_sp; };
    auto to_hz = [&](float mel) {
        return mel >= min_log_mel ? min_log_hz * expf(log_step * (mel - min_log_mel)) : f_sp * mel;
    };
    const float mel_lo = to_mel(0.0f), mel_hi = to_mel((float)sample_rate / 2.0f);
    std::vector<float> edge(n_mels + 2), freq(bins);
    for (int i = 0; i < n_mels + 2; ++i) edge[i] = to_hz(mel_lo + (float)i * (mel_hi - mel_lo) / (float)(n_mels + 1));
    for (int i = 0; i < bins; ++i) freq[i] = (float)i * (float)sample_rate / (float)n_fft;
    fb.assign((size_t)n_mels * bins, 0.0f);
    for (int m = 0; m < n_mels; ++m) {
        const float l = edge[m], c = edge[m + 1], r = edge[m + 2];
        const float norm = 2.0f / (r - l);
        for (int b = 0; b < bins; ++b) {
            const float f = freq[b];
            if (f >= l && f < c) fb[(size_t)m * bins + b] = norm * (f - l) / (c - l);
            else if (f >= c && f <= r) fb[(size_t)m * bins + b] = norm * (r - f) / (r - c);
        }
    }
}

// Swift's min / max on Comparable: min(x, y) = y < x ? y : x, max(x, y) = y >= x ? y : x
template <typename T> static T swift_min(T x, T y) { return y < x ? y : x; }
template <typename T> static T swift_max(T x, T y) { return y >= x ? y : x; }

// CoherePipeline.swift:90-97: symmetric Hann, and a length-1 window is [0] (build_window would divide by zero)
static void build_window_cohere(int length, std::vector<float> &w) {
    if (length > 1) build_window(length, false, w);
    else w.assign(length, 0.0f);
}

// CoherePipeline.swift:273-323 (slaneyMelFilter): Float32 throughout, f_min .. f_max, 1e-10 clamped denominators
static void build_filterbank_cohere(int n_fft, int n_mels, int sample_rate, float f_min, float f_max,
                                    std::vector<float> &fb) {
    const int bins = n_fft / 2 + 1;
    const float f_sp = 200.0f / 3.0f, min_log_hz = 1000.0f, min_log_mel = 15.0f, log_step = 0.06875177742f;
    auto to_mel = [&](float hz) { return hz >= min_log_hz ? min_log_mel + logf(hz / min_log_hz) / log_step : hz / f_sp; };
    auto to_hz = [&](float mel) {
        return mel >= min_log_mel ? min_log_hz * expf(log_step * (mel - min_log_mel)) : f_sp * mel;
    };
    std::vector<float> freq(bins), hz(n_mels + 2);
    for (int k = 0; k < bins; ++k) freq[k] = (float)sample_rate * (float)k / (float)n_fft;
    const float mel_min = to_mel(f_min), mel_max = to_mel(f_max);
    const float step = (mel_max - mel_min) / (float)(n_mels + 1);
    for (int i = 0; i < n_mels + 2; ++i) hz[i] = to_hz(mel_min + (float)i * step);
    fb.assign((size_t)n_mels * bins, 0.0f);
    for (int m = 0; m < n_mels; ++m) {
        const float lower = hz[m], center = hz[m + 1], upper = hz[m + 2];
        const float left_den = swift_max(center - lower, 1e-10f), right_den = swift_max(upper - center, 1e-10f);
        float *row = &fb[(size_t)m * bins];
        for (int k = 0; k < bins; ++k) {
            const float f = freq[k];
            if (f < lower || f > upper) continue;
            row[k] = f <= center ? (f - lower) / left_den : (upper - f) / right_den;
        }
        const float enorm = 2.0f / swift_max(upper - lower, 1e-10f);
        for (int k = 0; k < bins; ++k) row[k] *= enorm;
    }
}

// StyleTTS2MelExtractor.swift:160-221 (htkMelFilterbank): HTK scale in Float32 (log10f, powf), no norm, 0 .. sr/2, bin
// frequencies k * (sr / nFFT) for the rate the table is built for (16 kHz for StyleTTS2's 24 kHz audio)
static void build_filterbank_htk_f32(int n_fft, int n_mels, int sample_rate, std::vector<float> &fb) {
    const int bins = n_fft / 2 + 1;
    auto to_mel = [](float hz) { return 2595.0f * log10f(1.0f + hz / 700.0f); };
    auto to_hz = [](float mel) { return 700.0f * (powf(10.0f, mel / 2595.0f) - 1.0f); };
    std::vector<float> freq(bins), hz(n_mels + 2);
    const float bin_step = (float)sample_rate / (float)n_fft;
    for (int k = 0; k < bins; ++k) freq[k] = (float)k * bin_step;
    const float mel_min = to_mel(0.0f), mel_max = to_mel((float)sample_rate / 2.0f);
    for (int i = 0; i < n_mels + 2; ++i) {
        const float frac = (float)i / (float)(n_mels + 1);
        hz[i] = to_hz(mel_min + (mel_max - mel_min) * frac);
    }
    fb.assign((size_t)n_mels * bins, 0.0f);
    for (int m = 0; m < n_mels; ++m) {
        const float left = hz[m], center = hz[m + 1], right = hz[m + 2];
        const float left_slope = center - left, right_slope = right - center;
        for (int k = 0; k < bins; ++k) {
            const float f = freq[k];
            if (f < left || f > right) continue;
            float val;
            if (f <= center) val = left_slope > 0 ? (f - left) / left_slope : 0.0f;
            else val = right_slope > 0 ? (right - f) / right_slope : 0.0f;
            fb[(size_t)m * bins + k] = swift_max(val, 0.0f);
        }
    }
}

// LuxTtsMelExtractor.swift:158-187 (torchaudio melscale_fbanks, norm nil, HTK): Double throughout, bins on
// linspace(0, sr/2, bins), Float(max(0, min(up, down)))
static void build_filterbank_htk_f64(int n_fft, int n_mels, int sample_rate, std::vector<float> &fb) {
    const int bins = n_fft / 2 + 1;
    const double f_max = (double)sample_rate / 2.0;
    auto to_mel = [](double hz) { return 2595.0 * log10(1.0 + hz / 700.0); };
    auto to_hz = [](double mel) { return 700.0 * (pow(10.0, mel / 2595.0) - 1.0); };
    const double mel_min = to_mel(0.0), mel_max = to_mel(f_max);
    std::vector<double> pts(n_mels + 2), freq(bins);
    for (int i = 0; i < n_mels + 2; ++i) pts[i] = to_hz(mel_min + (double)i * (mel_max - mel_min) / (double)(n_mels + 1));
    for (int b = 0; b < bins; ++b) freq[b] = (double)b * f_max / (double)(bins - 1);
    fb.assign((size_t)n_mels * bins, 0.0f);
    for (int m = 0; m < n_mels; ++m)
        for (int b = 0; b < bins; ++b) {
            const double up = (freq[b] - pts[m]) / (pts[m + 1] - pts[m]);
            const double down = (pts[m + 2] - freq[b]) / (pts[m + 2] - pts[m + 1]);
            fb[(size_t)m * bins + b] = (float)swift_max(0.0, swift_min(up, down));
        }
}

const char *check_ex_config(const MelConfig &c) {
    if (c.fb_kind < FA_MEL_FB_AUDIO_MEL || c.fb_kind > FA_MEL_FB_LUXTTS) return "filterbank must be one of FA_MEL_FB_* (0..3)";
    if (c.filter_sample_rate < 0) return "filter_sample_rate must be 0 (the audio's rate) or positive";
    if (c.center_edge != FA_MEL_EDGE_ZERO && c.center_edge != FA_MEL_EDGE_REFLECT)
        return "center_edge must be FA_MEL_EDGE_ZERO or FA_MEL_EDGE_REFLECT";
    if (!std::isfinite(c.spectrum_power) || !(c.spectrum_power > 0.0f)) return "spectrum_power must be finite and > 0";
    if (!std::isfinite(c.log_mean) || !std::isfinite(c.log_std) || c.log_std == 0.0f)
        return "log_mean must be finite and log_std finite and non-zero";
    if (!std::isfinite(c.f_min) || !std::isfinite(c.f_max)) return "f_min and f_max must be finite";
    if (c.fb_kind != FA_MEL_FB_COHERE && (c.f_min != 0.0f || (c.f_max > 0.0f && c.f_max != (float)c.filter_rate() / 2.0f)))
        return "f_min / f_max apply to FA_MEL_FB_COHERE only (the other tables span 0 .. filter_sample_rate / 2)";
    if (c.reflect() && c.preemph != 0.0f)
        return "FA_MEL_EDGE_REFLECT needs preemph 0 (no reference frontend pre-emphasises a reflected signal)";
    return nullptr;
}

void build_tables(const MelConfig &c, std::vector<float> &window, std::vector<float> &filterbank) {
    const int fr = c.filter_rate();
    if (c.fb_kind == FA_MEL_FB_COHERE && !c.window_periodic) build_window_cohere(c.win_length, window);
    else build_window(c.win_length, c.window_periodic != 0, window);
    switch (c.fb_kind) {
    case FA_MEL_FB_COHERE:
        build_filterbank_cohere(c.n_fft, c.n_mels, fr, c.f_min, c.f_max > 0.0f ? c.f_max : (float)fr / 2.0f, filterbank);
        break;
    case FA_MEL_FB_STYLETTS2: build_filterbank_htk_f32(c.n_fft, c.n_mels, fr, filterbank); break;
    case FA_MEL_FB_LUXTTS: build_filterbank_htk_f64(c.n_fft, c.n_mels, fr, filterbank); break;
    default: build_filterbank(c.n_fft, c.n_mels, fr, filterbank);
    }
}

MelBands pack_bands(const std::vector<float> &filterbank, int n_mels, int bins) {
    MelBands B;
    B.lo.resize(n_mels);
    B.hi.resize(n_mels);
    B.off.resize(n_mels);
    for (int m = 0; m < n_mels; ++m) {
        int a = bins, b = 0;
        for (int k = 0; k < bins; ++k)
            if (filterbank[(size_t)m * bins + k] != 0.0f) {
                a = std::min(a, k);
                b = k + 1;
            }
        if (b == 0) a = 0;
        a &= ~3;                       // whole bin quads: 16-byte aligned reads of the power row (pair rows, kPairStride)
        b = (b + 3) & ~3;              // may reach 260 > 257: the tile's pad columns are zero, so are these weights
        B.lo[m] = a;
        B.hi[m] = b;
        B.off[m] = B.nnz;              // a multiple of four: 16-byte aligned weight quads
        B.nnz += b - a;
    }
    // filterbank-stage schedule of mel512_kernel: groups of four consecutive filters, dealt to the kWarpsPerCta warps
    // longest first (cost = widest band of the group, in quads)
    const int groups = (n_mels + 3) / 4;
    std::vector<int> cost(groups, 0), order(groups);
    for (int g = 0; g < groups; ++g) {
        for (int m = 4 * g; m < std::min(n_mels, 4 * g + 4); ++m) cost[g] = std::max(cost[g], (B.hi[m] - B.lo[m]) >> 2);
        order[g] = g;
    }
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return cost[a] > cost[b]; });
    std::vector<std::vector<int>> mine(kWarpsPerCta);
    std::vector<long long> load(kWarpsPerCta, 0);
    // warp 0's lane 0 also computes the next tile's geometry and issues its bulk copy in this phase: measured, that is
    // worth more than a full share of the filterbank work (handicap 0 / 6 / 12 / 24 quads: 0.3109 / 0.3049 / 0.2996 /
    // 0.2982 ms per audio-hour, identical output; profiles/r02_mel.md), so warp 0 only takes a group when the others
    // are this far ahead
    load[0] = 24;
    for (int g : order) {
        int best = 0;
        for (int wv = 1; wv < kWarpsPerCta; ++wv)
            if (load[wv] + 2 * (long long)mine[wv].size() < load[best] + 2 * (long long)mine[best].size()) best = wv;
        mine[best].push_back(g);
        load[best] += cost[g] + 4;   // + per-iteration control
    }
    size_t iters = 0;
    for (auto &v : mine) iters = std::max(iters, v.size());
    B.slots.assign(iters * kWarpsPerCta * 4, MelSlot{0, 0, 0, -1});
    for (int wv = 0; wv < kWarpsPerCta; ++wv)
        for (size_t it = 0; it < mine[wv].size(); ++it)
            for (int q = 0; q < 4; ++q) {
                const int m = 4 * mine[wv][it] + q;
                if (m < n_mels) B.slots[(it * kWarpsPerCta + wv) * 4 + q] = MelSlot{B.lo[m], (B.hi[m] - B.lo[m]) >> 2, B.off[m], m};
            }
    return B;
}

std::vector<float> pack_weights(const std::vector<float> &filterbank, const MelBands &b, int bins, bool swizzled,
                                float scale) {
    std::vector<float> w;
    w.reserve(b.nnz);
    for (size_t m = 0; m < b.lo.size(); ++m)
        for (int k = b.lo[m]; k < b.hi[m]; ++k) {
            const int src = swizzled ? pow_pos(k) : k;   // position k holds bin src: pow_pos is an involution
            w.push_back(src < bins ? scale * filterbank[m * bins + src] : 0.0f);
        }
    return w;
}

void place_window(const std::vector<float> &window, int n_fft, int off_w, std::vector<float> &win_tab,
                  std::vector<uint8_t> &in_tab) {
    win_tab.assign(n_fft, 0.0f);
    in_tab.assign(n_fft, 0);
    for (size_t j = 0; j < window.size(); ++j) {
        win_tab[off_w + j] = window[j];
        in_tab[off_w + j] = 1;
    }
}

} // namespace mel
} // namespace fa
