// Offline Sortformer window arithmetic (OfflineSortformerDiarizer.swift:98-119 and :279-375,
// SortformerSpeakerStitcher.swift:27-90), shared by the kernels (offline_sortformer_kernels.cu) and the host emulation
// of the CPU test-suite (tests/emul/offline_sortformer_emul.cpp).  Plain C++ under FA_HD: the host build compiles it
// with g++ -ffp-contract=off, the device build rounds every float operation separately through the _rn intrinsics.
#pragma once

#include "../fa_common.cuh"

#include <cstdint>

namespace fa {
namespace offline_sortformer {

constexpr int kWindowOut = 384;                        // windowOutputFrames
constexpr int kSubsampling = 8;                        // subsamplingFactor
constexpr int kWindowMel = kWindowOut * kSubsampling;  // windowMelFrames = 3072
constexpr int kSpeakers = 4;                           // numSpeakers
constexpr int kMels = 128;                             // melFeatures
constexpr int kPerms = 24;                             // 4!
constexpr int kDefaultOverlap = 100;                   // overlapOutputFrames

#if defined(__CUDA_ARCH__)
FA_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
FA_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
#else
FA_HD float fmul(float a, float b) { return a * b; }
FA_HD float fadd(float a, float b) { return a + b; }
#endif

// processComplete's overlapOut = max(0, min(overlapOutputFrames, windowOutputFrames - 1))
FA_HD int clamp_overlap(int overlap) { return overlap < 0 ? 0 : overlap > kWindowOut - 1 ? kWindowOut - 1 : overlap; }
FA_HD int hop_mel(int overlap) { return (kWindowOut - overlap) * kSubsampling; }

// totalOut = ceil(numMelFrames / subsampling)
FA_HD long long total_out(long long mel_frames) { return (mel_frames + kSubsampling - 1) / kSubsampling; }

// The windows of processComplete's `while melStart < numMelFrames` loop: window k starts at k * hopMel and the loop
// ends after the first window with fewer than windowMel frames.  The windows k * hop + 3072 <= n are full; the start
// after the last of them holds one more, partial window when it is still inside the file.
FA_HD long long window_count(long long mel_frames, int overlap) {
    if (mel_frames <= 0) return 0;
    if (mel_frames < kWindowMel) return 1;
    const long long hop = hop_mel(overlap);
    const long long full = (mel_frames - kWindowMel) / hop + 1;
    return full + (full * hop < mel_frames ? 1 : 0);
}

// Window k of a file of n mel frames: its first mel frame, validMel and validOut
struct Window {
    long long mel_start;
    int valid_mel, valid_out;
};
FA_HD Window window_at(long long n, int overlap, long long k) {
    Window w;
    w.mel_start = k * hop_mel(overlap);
    const long long left = n - w.mel_start;
    w.valid_mel = left < kWindowMel ? (int)left : kWindowMel;
    w.valid_out = (w.valid_mel + kSubsampling - 1) / kSubsampling;
    return w;
}

// The stitched overlap of a window at output frame g_start: min(overlap, validOut, max(0, totalOut - gStart))
FA_HD int overlap_frames(int overlap, int valid_out, long long total, long long g_start) {
    const long long room = total - g_start > 0 ? total - g_start : 0;
    long long ov = overlap < valid_out ? overlap : valid_out;
    return (int)(room < ov ? room : ov);
}

// Global speaker g's window column in permutation p, in the order of the stitcher's swap recursion (:80-90):
// 0123 0132 0213 0231 0321 0312 1023 1032 1203 1230 1320 1302 2103 2130 2013 2031 2301 2310 3120 3102 3210 3201 3021
// 3012, packed 2 bits per speaker, 8 permutations per word.
FA_HD int perm_at(int p, int g) {
    const uint64_t w = p < 8 ? 0xb1e19c6c78d8b4e4ull : p < 16 ? 0x72d236c68d2d39c9ull : 0x93634b1b87271e4eull;
    return (int)((w >> (8 * (p & 7) + 2 * g)) & 3);
}

// correlation[g][w] over `frames` staged overlap rows [frames x 4] of the global timeline and the window: one product
// and one sum per frame, each rounded, frames ascending, a frame skipped when the global value is +0 or -0 (NaN is not)
FA_HD float correlation(const float *global, const float *window, int frames, int g, int w) {
    float c = 0.0f;
    for (int f = 0; f < frames; ++f) {
        const float gv = global[f * kSpeakers + g];
        if (gv != 0.0f) c = fadd(c, fmul(gv, window[f * kSpeakers + w]));
    }
    return c;
}

// A permutation's score from its four correlations c[g][perm[g]], summed from 0 in speaker order
FA_HD float score(float c0, float c1, float c2, float c3) { return fadd(fadd(fadd(fadd(0.0f, c0), c1), c2), c3); }

// A filled frame's new value: (global + pred) * 0.5, the add then the multiply rounded
FA_HD float average(float global, float pred) { return fmul(fadd(global, pred), 0.5f); }

} // namespace offline_sortformer
} // namespace fa
