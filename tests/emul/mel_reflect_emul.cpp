// Host check of the any-nFFT kernel's reflect loader (FA_MEL_EDGE_REFLECT; CPU test-suite only).  Uses the kernel's own
// reflect_index (fluidaudio_b200/csrc/mel_core.cuh):
//   extern "C" void reflect_map(n, pad, idx[n + 2 pad])    the sample index each position of the padded clip reads
//   extern "C" void reflect_frames(x, n, n_fft, hop, win_tab[n_fft], in_tab[n_fft], T, out[T x n_fft])
//     the windowed float32 frames mel_generic_kernel<true, ...> hands its transform for a .center launch of T frames
#include "../../fluidaudio_b200/csrc/mel_core.cuh"

using namespace fa::mel;

extern "C" void reflect_map(long long n, int pad, long long *idx) {
    for (long long p = 0; p < n + 2 * pad; ++p) idx[p] = n > 0 ? reflect_index(p - pad, n) : -1;
}

extern "C" void reflect_frames(const float *x, long long n, int n_fft, int hop, const float *win_tab,
                               const unsigned char *in_tab, long long T, float *out) {
    const int pad = n_fft / 2;
    for (long long f = 0; f < T; ++f) {
        const long long base = f * hop - pad;
        for (int j = 0; j < n_fft; ++j) {
            float v = 0.0f;
            if (n > 0 && in_tab[j]) {
                const float a = x[reflect_index(base + j, n)], w = win_tab[j];
                v = a * w;
            }
            out[f * n_fft + j] = v;
        }
    }
}
