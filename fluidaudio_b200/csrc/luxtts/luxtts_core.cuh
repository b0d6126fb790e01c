// LuxTTS synthesis arithmetic (LuxTtsSynthesizer.swift:46-299, LuxTtsSolver.swift, StyleTTS2DiffusionSchedule.swift:45-81),
// shared by the kernels (luxtts_kernels.cu) and the host emulation of the CPU test-suite (tests/emul/luxtts_emul.cpp).
// Plain C++ under FA_HD: the host build compiles it with g++ -ffp-contract=off, the device build rounds every float
// product and sum separately through the _rn intrinsics.
#pragma once

#include "../fa_common.cuh"

#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>

namespace fa {
namespace luxtts {

constexpr int kFeat = 100;                // featDim
constexpr int kMaxFrames = 1024;          // maxFrames
constexpr int kSlotFloats = kMaxFrames * kFeat;
constexpr int kMaxTokens = 256;           // maxTokens
constexpr long long kMaxPrompt = 120000;  // Int(maxPromptSeconds 5.0 * melSampleRate 24000)
constexpr int kSteps = 4;                 // numSteps
constexpr int kHop = 256;                 // hopLength (24 kHz mel)
constexpr int kHop48k = 512;              // hop48k
constexpr int kBucketSmall = 282, kBucketLarge = 555;   // vocoderBuckets
constexpr int kRmsLanes = 256;            // lanes of the RMS tree
constexpr uint64_t kGamma = 0x9E3779B97F4A7C15ull;
constexpr uint64_t kSeedZero = 0xDEADBEEFCAFEBABEull;
constexpr double kTwoPi = 2.0 * 3.14159265358979311599796346854;   // 2.0 * Double.pi, exact

enum Reason : int {
    kOk = 0, kNoPromptTokens, kNoTextTokens, kNoPromptSamples, kBadSpeed, kSilent, kTooShort, kTooManyTokens,
    kTooLong, kTooFewFrames, kNoBucket, kDegenerate
};

#if defined(__CUDA_ARCH__)
FA_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
FA_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
FA_HD double dmul(double a, double b) { return __dmul_rn(a, b); }
FA_HD double dadd(double a, double b) { return __dadd_rn(a, b); }
FA_HD double ddiv(double a, double b) { return __ddiv_rn(a, b); }
#else
FA_HD float fmul(float a, float b) { return a * b; }
FA_HD float fadd(float a, float b) { return a + b; }
FA_HD double dmul(double a, double b) { return a * b; }
FA_HD double dadd(double a, double b) { return a + b; }
FA_HD double ddiv(double a, double b) { return a / b; }
#endif

// ------------------------------------------------------------------------------------------------ noise
FA_HD uint64_t seed_state(uint64_t seed) { return seed == 0 ? kSeedZero : seed; }

// The uniform of draw k >= 1: SplitMix64's output for state s0 + k * gamma, mapped to (0, 1].
FA_HD double uniform_at(uint64_t s0, uint64_t k) {
    uint64_t z = s0 + k * kGamma;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    const double u = ddiv((double)(z >> 11), 9007199254740992.0);
    return u <= 0 ? DBL_MIN : u;
}

// Gaussian j of the stream: nextGaussian() after j earlier calls, which read draws 2j + 1 and 2j + 2.
FA_HD float gaussian_at(uint64_t s0, uint64_t j) {
    const double u1 = uniform_at(s0, 2 * j + 1), u2 = uniform_at(s0, 2 * j + 2);
#if defined(__CUDA_ARCH__)
    const double mag = __dsqrt_rn(dmul(-2.0, log(u1)));
#else
    const double mag = std::sqrt(dmul(-2.0, std::log(u1)));
#endif
    return (float)dmul(mag, cos(dmul(kTwoPi, u2)));
}

// ------------------------------------------------------------------------------------------------ solver
// LuxTtsSolver.timeSteps(numSteps: 4, tShift: 0.5)[i] in float64
FA_HD double time_step(int i) {
    const double u = ddiv((double)i, (double)kSteps);
    return ddiv(dmul(0.5, u), dadd(1.0, dmul(0.5 - 1.0, u)));
}

// One float32 anchor-Euler update of element x with velocity v at t = tc, next tn (vDSP_vsma / vDSP_vsmsma).
FA_HD float anchor_euler(float x, float v, float tc, float tn, bool last) {
    const float x1p = fadd(fmul(v, 1.0f - tc), x);
    if (last) return x1p;
    const float x0p = fadd(fmul(v, -tc), x);
    return fadd(fmul(x0p, 1.0f - tn), fmul(x1p, tn));
}

// tokensIndex[f] for avg = features_length / token_count >= 1: token f / avg for f < token_count * avg, else the pad slot
FA_HD int token_index(int f, int token_count, int avg) { return f < token_count * avg ? f / avg : token_count; }

// vDSP_vclip(-1, 1): NaN passes through
FA_HD float clip_unit(float x) { return x < -1.0f ? -1.0f : x > 1.0f ? 1.0f : x; }

// ------------------------------------------------------------------------------------------------ RMS
// Lane l's partial sum of squares: samples l, l + 256, ... in order, in float64 (each square is exact).
FA_HD double rms_lane(const float *x, long long n, int lane) {
    double s = 0.0;
    for (long long i = lane; i < n; i += kRmsLanes) s = dadd(s, dmul((double)x[i], (double)x[i]));
    return s;
}

// sqrtf(Float(sum / n)) of the tree's total
FA_HD float rms_of(double sum, long long n) {
#if defined(__CUDA_ARCH__)
    return __fsqrt_rn(__double2float_rn(ddiv(sum, (double)n)));
#else
    return std::sqrt((float)(sum / (double)n));
#endif
}

#if !defined(__CUDA_ARCH__)
// The kernel's tree on the host: the lanes' partials, then halving strides 128, 64, ..., 1.
inline float rms_tree(const float *x, long long n) {
    double p[kRmsLanes];
    for (int l = 0; l < kRmsLanes; ++l) p[l] = rms_lane(x, n, l);
    for (int s = kRmsLanes / 2; s > 0; s >>= 1)
        for (int l = 0; l < s; ++l) p[l] = p[l] + p[l + s];
    return rms_of(p[0], n);
}
#endif

// ------------------------------------------------------------------------------------------------ plan
struct Plan {
    int reason;
    int prompt_samples, prompt_frames, token_count, features_length, gen_frames, bucket;
};

// synthesize's guards up to tokensIndex, less the silent-prompt check (which needs the RMS)
inline Plan plan_request(long long samples, int prompt_tokens, int text_tokens, float speed) {
    Plan p{};
    if (prompt_tokens <= 0) return p.reason = kNoPromptTokens, p;
    if (text_tokens <= 0) return p.reason = kNoTextTokens, p;
    if (samples <= 0) return p.reason = kNoPromptSamples, p;
    if (!(speed > 0)) return p.reason = kBadSpeed, p;
    p.prompt_samples = (int)(samples < kMaxPrompt ? samples : kMaxPrompt);
    p.prompt_frames = (p.prompt_samples + kHop / 2) / kHop;   // lhotse's count: 0 below 128 samples
    if (p.prompt_frames <= 0) return p.reason = kTooShort, p;
    if ((long long)prompt_tokens + text_tokens + 1 > kMaxTokens) return p.reason = kTooManyTokens, p;
    p.token_count = prompt_tokens + text_tokens;
    // Double(P) / Double(pt) * Double(tt) / speed, rounded up; Int() traps from 2^63 on, and so does P + Int(..)
    const double g = std::ceil((double)p.prompt_frames / (double)prompt_tokens * (double)text_tokens / (double)speed);
    if (!(g < 9223372036854775808.0) || (long long)g > LLONG_MAX - p.prompt_frames || (long long)g + p.prompt_frames > kMaxFrames)
        return p.reason = kTooLong, p;
    p.features_length = p.prompt_frames + (int)g;
    p.gen_frames = (int)g;
    if (p.gen_frames < 2) return p.reason = kTooFewFrames, p;
    p.bucket = p.gen_frames <= kBucketSmall ? kBucketSmall : p.gen_frames <= kBucketLarge ? kBucketLarge : 0;
    if (!p.bucket) return p.reason = kNoBucket, p;
    if (p.features_length / p.token_count < 1) return p.reason = kDegenerate, p;
    return p;
}

} // namespace luxtts
} // namespace fa
