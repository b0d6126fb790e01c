// Host tables of the log-mel plan: the configuration, the window and filterbank each reference class builds, and the
// packed form the kernels read the filterbank in (mel_tables.cpp).  Plain C++: no CUDA runtime call and no CUDA type, so
// the CPU test-suite compiles it with g++ (tests/emul/mel_tables_shim.cpp).
#pragma once

#include "fluidaudio_b200.h"
#include <cstdint>
#include <vector>

namespace fa {
namespace mel {

// Mirrors the parameters of AudioMelSpectrogram.init (AudioMelSpectrogram.swift:59-70).
struct MelConfig {
    int32_t sample_rate;
    int32_t n_mels;
    int32_t n_fft;
    int32_t hop_length;
    int32_t win_length;
    float preemph;
    int32_t pad_to;
    float log_floor;
    int32_t log_floor_mode;    // 0 additive log(x + floor), 1 clamped log(max(x, floor))
    int32_t window_periodic;
    // fa_mel_ex_config (fa_mel_create_ex); the defaults are fa_mel_create's behaviour
    int32_t fb_kind = FA_MEL_FB_AUDIO_MEL;      // FA_MEL_FB_*
    int32_t filter_sample_rate = 0;             // 0 = sample_rate
    float f_min = 0.0f, f_max = 0.0f;
    int32_t center_edge = FA_MEL_EDGE_ZERO;     // FA_MEL_EDGE_*
    float spectrum_power = 2.0f;
    float log_mean = 0.0f, log_std = 1.0f;

    int filter_rate() const { return filter_sample_rate > 0 ? filter_sample_rate : sample_rate; }
    bool reflect() const { return center_edge == FA_MEL_EDGE_REFLECT; }
    bool affine() const { return log_mean != 0.0f || log_std != 1.0f; }
    // every ex field as fa_mel_create leaves it: the streams and the NeMo adapters accept only such handles
    bool neutral() const {
        return fb_kind == FA_MEL_FB_AUDIO_MEL && filter_rate() == sample_rate && f_min == 0.0f && f_max <= 0.0f &&
               center_edge == FA_MEL_EDGE_ZERO && spectrum_power == 2.0f && !affine();
    }
};

// Spectrum the any-nFFT kernel feeds its filterbank: |X|^2 (the power tile holds 4|X|^2, the weights carry 1/4),
// |X| or |X|^p (the tile holds the value itself, the weights are unscaled).
enum { kSpecPower = 0, kSpecMagnitude = 1, kSpecGeneral = 2 };
inline int spectrum_kind(float p) { return p == 2.0f ? kSpecPower : (p == 1.0f ? kSpecMagnitude : kSpecGeneral); }

// Every fa_mel_ex_config field the kernels cannot honour: the reason as text, or nullptr when the config is fine.
const char *check_ex_config(const MelConfig &c);

// The window [win_length] and the dense filterbank [n_mels x (n_fft/2 + 1)] of c.fb_kind, each restating its Swift in
// that Swift's arithmetic, as the reference exposes them (getFilterbank).
void build_tables(const MelConfig &c, std::vector<float> &window, std::vector<float> &filterbank);

// One slot of mel512_kernel's filterbank schedule, in int4's member order (the device copy is an int4 array).
struct MelSlot {
    int lo;      // first bin
    int quads;   // bin quads of the band
    int off;     // offset of its packed weights
    int mel;     // mel bin, -1 for an empty slot
};

// Banded filterbank: per mel the contiguous range of non-zero bins [lo, hi), widened with explicit zero weights to whole
// bin quads, its weights packed at off (the prefix sum of the band widths, so every band starts 16-byte aligned).
struct MelBands {
    std::vector<int> lo, hi, off;
    int nnz = 0;                  // packed weights
    std::vector<MelSlot> slots;   // mel512_kernel's schedule: slot = (iteration * kWarpsPerCta + warp) * 4 + member
};
MelBands pack_bands(const std::vector<float> &filterbank, int n_mels, int bins);

// The band weights times `scale`, packed in the order the kernel finds the bins in its power tile: swizzled inside each
// bin quad (pow_pos, mel_core.cuh) for mel512_kernel, natural order for mel_generic_kernel.
std::vector<float> pack_weights(const std::vector<float> &filterbank, const MelBands &b, int bins, bool swizzled,
                                float scale);

// The window at offset off_w of an n_fft frame (win_tab), and which frame positions it covers (in_tab).
void place_window(const std::vector<float> &window, int n_fft, int off_w, std::vector<float> &win_tab,
                  std::vector<uint8_t> &in_tab);

} // namespace mel
} // namespace fa
