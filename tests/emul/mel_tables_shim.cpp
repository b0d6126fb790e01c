// C entry points over the log-mel plan's host tables (fluidaudio_b200/csrc/mel_tables.cpp, compiled with this file by
// g++): the window and filterbank of every kind, the packed filterbank and schedule, the window placement and the ex
// config check, for tests/test_mel_tables.py.
#include "mel_core.cuh"
#include "mel_tables.h"

#include <algorithm>
#include <cstring>

using namespace fa::mel;

static MelConfig config(int sample_rate, int n_mels, int n_fft, int win_length, int window_periodic, int fb_kind,
                        int filter_sample_rate, float f_min, float f_max) {
    MelConfig c{sample_rate, n_mels, n_fft, 160, win_length, 0.0f, 0, 5.9604645e-08f, 0, window_periodic};
    c.fb_kind = fb_kind;
    c.filter_sample_rate = filter_sample_rate;
    c.f_min = f_min;
    c.f_max = f_max;
    return c;
}

extern "C" {

// window [win_length], filterbank [n_mels x (n_fft/2 + 1)]
void mt_tables(int sample_rate, int n_mels, int n_fft, int win_length, int window_periodic, int fb_kind,
               int filter_sample_rate, float f_min, float f_max, float *window, float *filterbank) {
    std::vector<float> w, fb;
    build_tables(config(sample_rate, n_mels, n_fft, win_length, window_periodic, fb_kind, filter_sample_rate, f_min,
                        f_max),
                 w, fb);
    std::copy(w.begin(), w.end(), window);
    std::copy(fb.begin(), fb.end(), filterbank);
}

// sizes of the packed form of a dense [n_mels x bins] filterbank: packed weights and schedule slots
void mt_pack_sizes(const float *filterbank, int n_mels, int bins, int *nnz, int *n_slots) {
    const MelBands b = pack_bands(std::vector<float>(filterbank, filterbank + (size_t)n_mels * bins), n_mels, bins);
    *nnz = b.nnz;
    *n_slots = (int)b.slots.size();
}

// lo / hi / off [n_mels], weights [nnz], slots [n_slots x 4]
void mt_pack(const float *filterbank, int n_mels, int bins, int swizzled, float scale, int *lo, int *hi, int *off,
             float *w, int *slots) {
    const std::vector<float> fb(filterbank, filterbank + (size_t)n_mels * bins);
    const MelBands b = pack_bands(fb, n_mels, bins);
    std::copy(b.lo.begin(), b.lo.end(), lo);
    std::copy(b.hi.begin(), b.hi.end(), hi);
    std::copy(b.off.begin(), b.off.end(), off);
    const std::vector<float> pw = pack_weights(fb, b, bins, swizzled != 0, scale);
    std::copy(pw.begin(), pw.end(), w);
    if (!b.slots.empty()) std::memcpy(slots, b.slots.data(), b.slots.size() * sizeof(MelSlot));
}

int mt_warps_per_cta() { return kWarpsPerCta; }

// win_tab / in_tab [n_fft]
void mt_place_window(const float *window, int win_length, int n_fft, int off_w, float *win_tab, uint8_t *in_tab) {
    std::vector<float> wt;
    std::vector<uint8_t> it;
    place_window(std::vector<float>(window, window + win_length), n_fft, off_w, wt, it);
    std::copy(wt.begin(), wt.end(), win_tab);
    std::copy(it.begin(), it.end(), in_tab);
}

// check_ex_config's reason, or null
const char *mt_check(int sample_rate, int fb_kind, int filter_sample_rate, float f_min, float f_max, int center_edge,
                     float preemph, float spectrum_power, float log_mean, float log_std) {
    MelConfig c = config(sample_rate, 80, 512, 400, 0, fb_kind, filter_sample_rate, f_min, f_max);
    c.center_edge = center_edge;
    c.preemph = preemph;
    c.spectrum_power = spectrum_power;
    c.log_mean = log_mean;
    c.log_std = log_std;
    return check_ex_config(c);
}

} // extern "C"
