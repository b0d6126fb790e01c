// Host run of StyleTTS2 synthesis glue arithmetic (fluidaudio_b200/csrc/styletts2/styletts2_core.cuh; CPU test-suite
// only), in the kernels' own formulation: the bucket, counter-based noise, the blend, one token's duration, and the
// fused expansion (prefix sums, token search, 0 + value) of one request.
#include "../../fluidaudio_b200/csrc/styletts2/styletts2_core.cuh"

#include <cstdint>
#include <vector>

using namespace fa::styletts2;

extern "C" {

int styletts2_emul_bucket(int token_count, int *reason) { return bucket_for(token_count, reason); }

void styletts2_emul_noise(uint64_t seed, int count, float *out) {
    for (int j = 0; j < count; ++j) out[j] = noise_at(seed, j);
}

void styletts2_emul_blend(const float *s_pred, const float *ref_s, float alpha, float beta, float *ref, float *s) {
    for (int k = 0; k < kRefSplit; ++k) {
        ref[k] = blend(alpha, s_pred[k], ref_s[k]);
        s[k] = blend(beta, s_pred[kRefSplit + k], ref_s[kRefSplit + k]);
    }
}

// durations [n] of logits [n x channels]; -1 for a NaN sum
void styletts2_emul_durations(const float *logits, int n, int channels, int *out) {
    for (int t = 0; t < n; ++t) out[t] = duration_of(logits + (int64_t)t * channels, channels);
}

// en [dC x frame_stride] and asr [tC x frame_stride] of one request from its durations, d [n x dC], t_en [tC x n]
void styletts2_emul_expand(const int *durations, int n, const float *d, int d_channels, const float *t_en,
                           int t_channels, int64_t frame_stride, float *en, float *asr) {
    std::vector<long long> starts((size_t)n + 1, 0);
    for (int t = 0; t < n; ++t) starts[(size_t)t + 1] = starts[(size_t)t] + durations[t];
    const long long F = starts[(size_t)n];
    for (int64_t f = 0; f < frame_stride; ++f) {
        const int tk = f < F ? token_at(starts.data(), n, f > 0 ? f - 1 : 0) : -1;
        for (int c = 0; c < d_channels; ++c)
            en[(int64_t)c * frame_stride + f] = tk >= 0 ? expanded(d[(int64_t)tk * d_channels + c]) : 0.0f;
        for (int c = 0; c < t_channels; ++c)
            asr[(int64_t)c * frame_stride + f] = tk >= 0 ? expanded(t_en[(int64_t)c * n + tk]) : 0.0f;
    }
}

} // extern "C"
