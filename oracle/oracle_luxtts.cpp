// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
//
// A sequential CPU restatement of LuxTtsSynthesizer.synthesize's host arithmetic (Sources/FluidAudio/TTS/LuxTts/
// LuxTtsSynthesizer.swift:46-299), LuxTtsSolver (LuxTtsSolver.swift) and StyleTTS2NoiseSource
// (TTS/StyleTTS2/Pipeline/Sampler/StyleTTS2DiffusionSchedule.swift:45-81), line by line in the reference's order.  The
// prompt mel is an input: LuxTtsMelExtractor has its own oracle (oracle_mel_torch.cpp).  Where vDSP leaves an order or
// a fusing open, this file takes the plain reading: the mean square sums in index order in float64, and every float32
// product and sum of the anchor-Euler update rounds separately.  Built with -O2 -ffp-contract=off on baseline x86-64.
#include <cfloat>
#include <cmath>
#include <cstdint>

namespace {

constexpr int kFeatDim = 100, kMaxFrames = 1024, kMaxTokens = 256, kNumSteps = 4, kHop48k = 512;
constexpr float kFeatScale = 0.1f, kTargetRms = 0.1f, kLogMelFloor = 1e-7f;
constexpr double kTShift = 0.5, kMaxPromptSeconds = 5.0;
constexpr int kMelSampleRate = 24000, kHop = 256;

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

double time_step(int i) {
    const double u = double(i) / double(kNumSteps);
    return kTShift * u / (1.0 + (kTShift - 1.0) * u);
}

} // namespace

extern "C" {

// synthesize's guards before the models, less the silent check; out = {prompt_samples, prompt_frames, token_count,
// features_length, gen_frames, bucket}.  Returns the reason code (fa_luxtts_plan_info.reason).
int oracle_luxtts_plan(int64_t samples, int32_t prompt_tokens, int32_t text_tokens, float speed, int32_t *out) {
    for (int i = 0; i < 6; ++i) out[i] = 0;
    if (prompt_tokens == 0) return 1;
    if (text_tokens == 0) return 2;
    if (samples == 0) return 3;
    if (!(speed > 0)) return 4;
    const int64_t max_prompt = int64_t(kMaxPromptSeconds * double(kMelSampleRate));
    const int64_t n = samples < max_prompt ? samples : max_prompt;
    out[0] = (int32_t)n;
    const int64_t prompt_frames = (n + kHop / 2) / kHop;   // LuxTtsMelExtractor.frameCount
    out[1] = (int32_t)prompt_frames;
    if (!(prompt_frames > 0)) return 6;
    const int64_t token_count = int64_t(prompt_tokens) + int64_t(text_tokens);
    if (!(token_count + 1 <= kMaxTokens)) return 7;
    out[2] = (int32_t)token_count;
    // LuxTtsSolver.featuresLength: Double(P) / Double(pt) * Double(tt) / speed, rounded up, then Int(); Swift traps
    // on a value Int cannot hold and on the overflowing sum, both refused here as too long
    const double generated = double(prompt_frames) / double(prompt_tokens) * double(text_tokens) / double(speed);
    const double up = std::ceil(generated);
    if (!(up >= -9223372036854775808.0 && up < 9223372036854775808.0)) return 8;
    const int64_t g = int64_t(up);
    if (g > INT64_MAX - prompt_frames) return 8;
    const int64_t features_length = prompt_frames + g;
    if (!(features_length <= kMaxFrames)) return 8;
    out[3] = (int32_t)features_length;
    const int64_t gen_frames = features_length - prompt_frames;
    out[4] = (int32_t)gen_frames;
    if (!(gen_frames >= 2)) return 9;
    const int buckets[2] = {282, 555};
    int bucket = 0;
    for (int b : buckets)
        if (b >= gen_frames) {
            bucket = b;
            break;
        }
    if (!bucket) return 10;
    out[5] = bucket;
    if (!(features_length / token_count >= 1)) return 11;   // LuxTtsSolver.tokensIndex
    return 0;
}

// vDSP_measqv then sqrt: the mean square summed in index order in float64, rounded once to float32
float oracle_luxtts_rms(const float *x, int64_t n) {
    double s = 0.0;
    for (int64_t i = 0; i < n; ++i) s += double(x[i]) * double(x[i]);
    const float mean_square = float(s / double(n));
    return std::sqrt(mean_square);
}

// the prompt after `if promptRms < targetRms { vDSP_vsmul(prompt, gain = targetRms / promptRms) }`
void oracle_luxtts_gain(const float *x, int64_t n, float rms, float *out) {
    const bool boost = rms < kTargetRms;
    const float gain = kTargetRms / rms;
    for (int64_t i = 0; i < n; ++i) out[i] = boost ? x[i] * gain : x[i];
}

// noise.nextGaussianArray(count:)
void oracle_luxtts_noise(uint64_t seed, int64_t count, float *out) {
    Noise noise(seed);
    for (int64_t i = 0; i < count; ++i) out[i] = noise.next_gaussian();
}

// the raw draws (SplitMix64 outputs) and their uniforms, for the counter-based checks
void oracle_luxtts_uniforms(uint64_t seed, int64_t count, double *out) {
    Noise noise(seed);
    for (int64_t i = 0; i < count; ++i) out[i] = noise.next_uniform();
}

void oracle_luxtts_time_steps(double *out) {
    for (int i = 0; i <= kNumSteps; ++i) out[i] = time_step(i);
}

// LuxTtsSolver.tokensIndex: 0, or -1 for the degenerate duration
int oracle_luxtts_tokens_index(int64_t tokens_count, int64_t features_length, int64_t *out) {
    const int64_t avg = features_length / tokens_count;
    if (!(avg >= 1)) return -1;
    for (int64_t f = 0; f < features_length; ++f) out[f] = tokens_count;
    int64_t frame = 0;
    for (int64_t token = 0; token < tokens_count; ++token)
        for (int64_t k = 0; k < avg; ++k) out[frame++] = token;
    return 0;
}

// LuxTtsSolver.anchorEulerUpdate (float64)
void oracle_luxtts_anchor_euler_f64(const double *x, const double *v, int64_t n, double t_cur, double t_next,
                                    int is_last, double *out) {
    for (int64_t i = 0; i < n; ++i) {
        const double x1p = x[i] + (1.0 - t_cur) * v[i];
        if (is_last) {
            out[i] = x1p;
            continue;
        }
        const double x0p = x[i] - t_cur * v[i];
        out[i] = (1.0 - t_next) * x0p + t_next * x1p;
    }
}

// Stage 3's step `step` over the active count: vDSP_vsma / vDSP_vsmsma in float32, in place on x
void oracle_luxtts_step(float *x, const float *v, int64_t active, int step) {
    const float t_cur = float(time_step(step));
    const float t_next = float(time_step(step + 1));
    const bool is_last = step == kNumSteps - 1;
    const float one_minus_t = 1.0f - t_cur;
    for (int64_t i = 0; i < active; ++i) {
        const float x1p = v[i] * one_minus_t + x[i];
        if (is_last) {
            x[i] = x1p;
            continue;
        }
        const float neg_t = -t_cur;
        const float x0p = v[i] * neg_t + x[i];
        const float w0 = 1.0f - t_next, w1 = t_next;
        x[i] = x0p * w0 + x1p * w1;
    }
}

// Stage 2: text_condition, speech_condition [1024 x 100] and the frame mask [1024] from the compact embeds
// [(token_count + 1) x 100] and the unscaled prompt mel [prompt_frames x 100].  0, or -1 for the degenerate duration.
int oracle_luxtts_conditions(const float *embeds, int64_t token_count, int64_t features_length, const float *prompt_mel,
                             int64_t prompt_frames, float *text_condition, float *speech_condition, float *frame_mask) {
    for (int64_t i = 0; i < int64_t(kMaxFrames) * kFeatDim; ++i) text_condition[i] = speech_condition[i] = 0.0f;
    for (int64_t i = 0; i < kMaxFrames; ++i) frame_mask[i] = 0.0f;
    int64_t index[kMaxFrames];
    if (oracle_luxtts_tokens_index(token_count, features_length, index) != 0) return -1;
    for (int64_t frame = 0; frame < features_length; ++frame) {
        const int64_t src = index[frame] * kFeatDim, dst = frame * kFeatDim;
        for (int d = 0; d < kFeatDim; ++d) text_condition[dst + d] = embeds[src + d];
    }
    for (int64_t frame = 0; frame < prompt_frames; ++frame)
        for (int d = 0; d < kFeatDim; ++d)
            speech_condition[frame * kFeatDim + d] = prompt_mel[frame * kFeatDim + d] * kFeatScale;
    for (int64_t i = features_length; i < kMaxFrames; ++i) frame_mask[i] = 1.0f;
    return 0;
}

// Stage 4's melInput [100 x bucket]
void oracle_luxtts_vocoder_input(const float *x, int64_t prompt_frames, int64_t gen_frames, int64_t bucket, float *out) {
    const float log_floor = std::log(kLogMelFloor);
    const float inv_scale = 1.0f / kFeatScale;
    for (int m = 0; m < kFeatDim; ++m) {
        const int64_t row = m * bucket;
        for (int64_t f = 0; f < gen_frames; ++f) out[row + f] = x[(prompt_frames + f) * kFeatDim + m] * inv_scale;
        for (int64_t f = gen_frames; f < bucket; ++f) out[row + f] = log_floor;
    }
}

// The tail of synthesize: truncate, vDSP_vclip (NaN passes through), rescale a boosted prompt's output.  Returns the
// sample count.
int64_t oracle_luxtts_finish(const float *audio, int64_t output_samples, int64_t gen_frames, float prompt_rms,
                             float *out) {
    const int64_t want = (gen_frames - 1) * kHop48k;
    const int64_t count = want < output_samples ? want : output_samples;
    const float lo = -1.0f, hi = 1.0f;
    for (int64_t i = 0; i < count; ++i) {
        const float a = audio[i];
        out[i] = a < lo ? lo : (a > hi ? hi : a);
    }
    if (prompt_rms < kTargetRms) {
        const float gain = prompt_rms / kTargetRms;
        for (int64_t i = 0; i < count; ++i) out[i] = out[i] * gain;
    }
    return count;
}

} // extern "C"
