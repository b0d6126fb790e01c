// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
//
// A sequential CPU restatement of StyleTTS2Synthesizer.synthesize's glue between its models (Sources/FluidAudio/TTS/
// StyleTTS2/Pipeline/Synthesize/StyleTTS2Synthesizer.swift:33-133 and StyleTTS2GlueOps.swift:23-161) and of
// StyleTTS2NoiseSource (Pipeline/Sampler/StyleTTS2DiffusionSchedule.swift:45-81), line by line in the reference's
// order.  Where the reference calls a closed library this file takes a stated reading: expf is the correctly rounded
// float32 exp of oracle_float.h; cblas_sgemm is netlib's loop (C zeroed for beta = 0, then for each column j and each l with
// B(l, j) != 0, C(:, j) += (alpha B(l, j)) A(:, l)); vDSP_mtrans is the plain copy.  Built with -O2
// -ffp-contract=off on baseline x86-64.
#include <cfloat>
#include <cmath>
#include <cstdint>

#include "oracle_float.h"

namespace {

constexpr int kStyleDim = 256, kRefSplit = 128, kDiffusionSteps = 5, kDefaultBertTokens = 57, kTailTrim = 50;
constexpr int kBuckets[3] = {64, 128, 256};

// StyleTTS2NoiseSource
struct Noise {
    uint64_t state;
    explicit Noise(uint64_t seed) : state(seed == 0 ? 0xdeadbeefcafebabeull : seed) {}
    double next_uniform() {
        state += 0x9E3779B97F4A7C15ull;
        uint64_t z = state;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        z = z ^ (z >> 31);
        const double u = double(z >> 11) / double(1ull << 53);
        return u <= 0 ? DBL_MIN : u;
    }
    float next_gaussian() {
        const double u1 = next_uniform();
        const double u2 = next_uniform();
        const double mag = std::sqrt(-2.0 * std::log(u1));
        return float(mag * std::cos(2.0 * M_PI * u2));
    }
};

float expf_pinned(float x) { return oracle_float::exp32(x); }

} // namespace

extern "C" {

// synthesize's bucket choice and resolveBucket: the bucket, or 0 with *reason 1 (no token: synthesize would divide by
// realN = 0 at :59) or 2 (noBucketAvailable)
int oracle_styletts2_bucket(int64_t token_count, int32_t *reason) {
    *reason = 0;
    if (token_count == 0) return *reason = 1, 0;
    if (token_count <= kDefaultBertTokens) return kDefaultBertTokens;
    for (int size : kBuckets)
        if (token_count <= size) return size;
    return *reason = 2, 0;
}

// runBert's padded tokens and attention mask, and runFusedSampler's noise_init [256] then noises_aux [4 x 256]
void oracle_styletts2_sampler_inputs(const int32_t *ids, int64_t real_n, int64_t padded_t, uint64_t seed,
                                     int32_t *tokens, int32_t *mask, float *noise_init, float *noises_aux) {
    for (int64_t t = 0; t < real_n; ++t) tokens[t] = ids[t];
    for (int64_t t = real_n; t < padded_t; ++t) tokens[t] = 0;
    for (int64_t t = 0; t < real_n; ++t) mask[t] = 1;
    for (int64_t t = real_n; t < padded_t; ++t) mask[t] = 0;
    Noise rng(seed);
    for (int i = 0; i < kStyleDim; ++i) noise_init[i] = rng.next_gaussian();
    for (int s = 0; s < kDiffusionSteps - 1; ++s) {
        float row[kStyleDim];
        for (int i = 0; i < kStyleDim; ++i) row[i] = rng.next_gaussian();
        for (int i = 0; i < kStyleDim; ++i) noises_aux[s * kStyleDim + i] = row[i];
    }
}

// noise.nextGaussianArray(count:)
void oracle_styletts2_noise(uint64_t seed, int64_t count, float *out) {
    Noise rng(seed);
    for (int64_t i = 0; i < count; ++i) out[i] = rng.next_gaussian();
}

// roundDurations over logits [real_n x channels]: 0, or -1 where Int(NaN) traps
int oracle_styletts2_round_durations(const float *logits, int64_t real_n, int64_t channels, int64_t *durations) {
    for (int64_t t = 0; t < real_n; ++t) {
        float sum = 0;
        for (int64_t c = 0; c < channels; ++c) {
            const float x = logits[t * channels + c];
            sum += 1.0f / (1.0f + expf_pinned(-x));
        }
        if (std::isnan(sum)) return -1;
        const int64_t rounded = int64_t(std::round(sum));
        durations[t] = rounded > 1 ? rounded : 1;
    }
    return 0;
}

int64_t oracle_styletts2_total_frames(const int64_t *durations, int64_t real_n) {
    int64_t total = 0;
    for (int64_t i = 0; i < real_n; ++i) total += durations[i];
    return total;
}

// buildAlignmentMatrix: [real_n x total_frames]
void oracle_styletts2_alignment(const int64_t *durations, int64_t real_n, int64_t total_frames, float *matrix) {
    for (int64_t i = 0; i < real_n * total_frames; ++i) matrix[i] = 0;
    int64_t col = 0;
    for (int64_t i = 0; i < real_n; ++i) {
        const int64_t d = durations[i];
        for (int64_t k = 0; k < d; ++k) matrix[i * total_frames + col + k] = 1;
        col += d;
    }
}

// matmulAligned: out [channels x total_frames] = features [channels x real_n] @ alignment, netlib's loop
void oracle_styletts2_matmul_aligned(const float *features, int64_t channels, int64_t real_n, const float *alignment,
                                     int64_t total_frames, float *out) {
    const float alpha = 1.0f;
    for (int64_t j = 0; j < total_frames; ++j) {
        for (int64_t i = 0; i < channels; ++i) out[i * total_frames + j] = 0.0f;
        for (int64_t l = 0; l < real_n; ++l) {
            const float b = alignment[l * total_frames + j];
            if (b == 0.0f) continue;
            const float temp = alpha * b;
            for (int64_t i = 0; i < channels; ++i) out[i * total_frames + j] += temp * features[i * real_n + l];
        }
    }
}

// transposeLast2D: [rows x cols] -> [cols x rows]
void oracle_styletts2_transpose(const float *src, int64_t rows, int64_t cols, float *out) {
    for (int64_t r = 0; r < rows; ++r)
        for (int64_t c = 0; c < cols; ++c) out[c * rows + r] = src[r * cols + c];
}

// hifiganShift on [channels x frames]
void oracle_styletts2_hifigan_shift(const float *x, int64_t channels, int64_t frames, float *out) {
    for (int64_t c = 0; c < channels; ++c) {
        const int64_t row = c * frames;
        out[row] = x[row];
        for (int64_t f = 1; f < frames; ++f) out[row + f] = x[row + f - 1];
    }
}

// blendStyle
void oracle_styletts2_blend(const float *s_pred, const float *ref_s, float alpha, float beta, float *ref, float *s) {
    const float one_minus_alpha = 1.0f - alpha;
    const float one_minus_beta = 1.0f - beta;
    for (int i = 0; i < kRefSplit; ++i) {
        ref[i] = alpha * s_pred[i] + one_minus_alpha * ref_s[i];
        s[i] = beta * s_pred[kRefSplit + i] + one_minus_beta * ref_s[kRefSplit + i];
    }
}

// the tail trim: the samples synthesize keeps of `count`
int64_t oracle_styletts2_trim(int64_t count) {
    const int64_t trim = kTailTrim < count ? kTailTrim : count;
    return trim > 0 ? count - trim : count;
}

} // extern "C"
