// StyleTTS2 synthesis glue arithmetic (StyleTTS2Synthesizer.swift:33-133, StyleTTS2GlueOps.swift:23-161), shared by
// the kernels (styletts2_kernels.cu) and the host emulation of the CPU test-suite (tests/emul/styletts2_emul.cpp).
// Plain C++ under FA_HD: the host build compiles it with g++ -ffp-contract=off, the device build rounds every float
// operation separately through the _rn intrinsics.  The noise source is LuxTTS's (luxtts_core.cuh), which is
// StyleTTS2NoiseSource itself.
#pragma once

#include "../fa_float.cuh"
#include "../luxtts/luxtts_core.cuh"

#include <cmath>
#include <cstdint>

namespace fa {
namespace styletts2 {

constexpr int kStyleDim = 256;      // styleDim
constexpr int kRefSplit = 128;      // refSplit
constexpr int kNoiseRows = 5;       // diffusionSteps: noise_init and 4 noises_aux
constexpr int kNoiseFloats = kNoiseRows * kStyleDim;
constexpr int kDefaultTokens = 57;  // defaultBertTokens
constexpr int kMaxTokens = 256;     // the largest of bucketTokenSizes
constexpr int kTailTrim = 50;       // tailTrimSamples

enum Reason : int { kOk = 0, kNoTokens = 1, kNoBucket = 2, kNonfiniteDuration = 3 };

#if defined(__CUDA_ARCH__)
FA_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
FA_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
FA_HD float fsub(float a, float b) { return __fsub_rn(a, b); }
FA_HD float fdiv(float a, float b) { return __fdiv_rn(a, b); }
#else
FA_HD float fmul(float a, float b) { return a * b; }
FA_HD float fadd(float a, float b) { return a + b; }
FA_HD float fsub(float a, float b) { return a - b; }
FA_HD float fdiv(float a, float b) { return a / b; }
#endif

// resolveBucket with the default 57-token model in front: 57, 64, 128 or 256 (0 with a reason otherwise)
FA_HD int bucket_for(int token_count, int *reason) {
    *reason = kOk;
    if (token_count <= 0) return *reason = kNoTokens, 0;
    if (token_count <= kDefaultTokens) return kDefaultTokens;
    if (token_count <= 64) return 64;
    if (token_count <= 128) return 128;
    if (token_count <= kMaxTokens) return kMaxTokens;
    return *reason = kNoBucket, 0;
}

// Gaussian j of request's noise block [5 x 256]: nextGaussian() after j earlier draws of StyleTTS2NoiseSource(seed)
FA_HD float noise_at(uint64_t seed, int j) { return luxtts::gaussian_at(luxtts::seed_state(seed), (uint64_t)j); }

// blendStyle, one element: w * p + (1 - w) * r, 1 - w in float32, each product and sum rounded separately
FA_HD float blend(float w, float p, float r) { return fadd(fmul(w, p), fmul(fsub(1.0f, w), r)); }

// roundDurations for one token: the float32 sum of 1 / (1 + expf(-x)) over its C logits in channel order, expf the
// correctly rounded f_exp, rounded half away from zero, at least 1.  A NaN sum (any NaN logit) returns -1: Swift's Int(NaN) traps.
FA_HD int duration_of(const float *logits, int channels) {
    float sum = 0.0f;
    for (int c = 0; c < channels; ++c) sum = fadd(sum, fdiv(1.0f, fadd(1.0f, fp::f_exp(-logits[c]))));
    if (sum != sum) return -1;
    const int r = (int)roundf(sum);
    return r < 1 ? 1 : r;
}

// The token whose prefix interval holds frame g: the largest t < n with starts[t] <= g (starts[0] = 0, increasing)
FA_HD int token_at(const long long *starts, int n, long long g) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (starts[mid] <= g) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// One element of the expanded, shifted features: netlib sgemm with beta = 0 leaves 0 + 1 * v, so -0 becomes +0
FA_HD float expanded(float v) { return fadd(0.0f, v); }

} // namespace styletts2
} // namespace fa
