// Per-element arithmetic of the offline diarizer's prepare stage (prepare_kernels.cu), host- and device-callable so that
// the CPU suite runs the very code the kernels run (tests/emul/prepare_emul.cpp).
//
// Reference (paths under Sources/FluidAudio/Diarizer/Offline):
//   Segmentation/OfflineSegmentationProcessor.swift:15-24,321-405   per-frame powerset decoding
//   Utils/VDSPOperations.swift:142-155                              logSumExp
//   Extraction/WeightInterpolation.swift:19-146                     half-pixel linear interpolation
//   Extraction/OfflineEmbeddingExtractor.swift:381-387,421-613      per-speaker mask decisions, times
//   Extraction/OfflineEmbeddingExtractor.swift:835-842              maskCosineSimilarity
//
// Every float32 / float64 operation the reference states is one round-to-nearest operation here: the f_* / d_* helpers
// are the __f*_rn / __d*_rn intrinsics on the device (never contracted into an FMA) and the plain operators on the host,
// whose build keeps contraction off.  Swift's min / max are restated as the comparisons they are, so a NaN takes the
// branch it takes there.
#pragma once

#include "fa_common.cuh"
#include "fa_float.cuh"

#include <cfloat>
#include <cmath>

namespace fa {
namespace prepare {

constexpr int kPowersetClasses = 8;    // powerset.count: {}, {0}, {1}, {2}, {0,1}, {0,2}, {1,2}, {0,1,2}
constexpr int kDecodeSpeakers = 3;     // speakerCount of OfflineSegmentationProcessor
constexpr float kActiveThreshold = 1e-3f;   // overlapThreshold (:306), also first / last active frame (:587-588)
constexpr float kMinActiveRatio = 0.2f;     // minActiveRatio (:519)
constexpr int kSumLanes = 256;         // lanes of ordered_sum, = threads of a mask CTA

using namespace fa::fp;   // f_* / d_* and swift_min / swift_max (fa_float.cuh)

// Speakers of powerset class k as a bit mask (bit s = local speaker s).
FA_HD unsigned powerset_speakers(int k) {
    return k < 4 ? (k == 0 ? 0u : 1u << (k - 1)) : (k == 4 ? 3u : k == 5 ? 5u : k == 6 ? 6u : 7u);
}

struct FrameDecision {
    int best;     // argmax over the classes: strict >, from -greatestFiniteMagnitude, first wins (:327-335)
    int speech;   // clamp(1 - exp(logProb[0]), 0, 1) >= speechOnsetThreshold (:401-404)
};

// One frame: x[classes] logits in, logp[classes] = x + (-logSumExp(x)) out (:337-346); logp may alias x.  The sum of the
// shifted exponentials runs in class order (vDSP_sve's order is closed; so are vvexpf's bits, see DESIGN §2), and exp
// and log are the correctly rounded f_exp / f_log.
FA_HD FrameDecision decode_frame(const float *x, int classes, float onset, float *logp) {
    FrameDecision d;
    d.best = 0;
    float best = -FLT_MAX;
    for (int c = 0; c < classes; ++c)
        if (x[c] > best) {
            best = x[c];
            d.best = c;
        }
    float m = x[0];                                  // Sequence.max(): replaced while m < x[c]
    for (int c = 1; c < classes; ++c)
        if (m < x[c]) m = x[c];
    const float shift = -m;
    float sum = 0.0f;
    for (int c = 0; c < classes; ++c) sum = f_add(sum, f_exp(f_add(x[c], shift)));
    const float neg_lse = -f_add(f_log(sum), m);
    const float empty = f_exp(f_add(x[0], neg_lse));  // probabilityBuffer[emptyClassIndex]
    for (int c = 0; c < classes; ++c) logp[c] = f_add(x[c], neg_lse);
    const float speech = swift_max(0.0f, swift_min(1.0f, f_sub(1.0f, empty)));
    d.speech = speech >= onset ? 1 : 0;
    return d;
}

// WeightInterpolation.InterpolationCoefficients.init (:28-49) for output index i.
struct Interp {
    int left, right;
    float w_left, w_right;
};
FA_HD Interp interp_coefficients(int i, int in_len, int out_len) {
    const float scale = f_div((float)out_len, (float)in_len);
    const float position = f_sub(f_div(f_add((float)i, 0.5f), scale), 0.5f);
    const float clamped = swift_min(swift_max(position, 0.0f), (float)(in_len - 1));
    Interp k;
    k.left = (int)floorf(clamped);
    k.right = k.left + 1 < in_len - 1 ? k.left + 1 : in_len - 1;
    k.w_right = f_sub(clamped, (float)k.left);
    k.w_left = f_sub(1.0f, k.w_right);
    return k;
}
// WeightInterpolation.resample (:100-115), element i of the output: the input itself when the lengths match.
FA_HD float resample_at(const float *in, int in_len, int out_len, int i) {
    if (in_len == out_len) return in[i];
    const Interp k = interp_coefficients(i, in_len, out_len);
    return f_add(f_mul(in[k.left], k.w_left), f_mul(in[k.right], k.w_right));
}

// processChunk's decisions for one local speaker from the sums of its base and clean masks (:504-542).
struct MaskDecision {
    int candidate;   // goes on to be resampled (it is still dropped when its resampled energy is <= 0, :549)
    int use_clean;   // maskToUse = cleanMask (else baseMask)
    int fallback;    // fallbackMaskCount += 1
    float mask_sum;
};
FA_HD MaskDecision mask_decide(float base_sum, float clean_sum, int frames, int min_frames) {
    MaskDecision d = {0, 0, 0, 0.0f};
    if (base_sum <= 0.0f) return d;
    if (clean_sum < f_mul((float)frames, kMinActiveRatio)) return d;
    if (clean_sum >= (float)min_frames) {
        d.use_clean = 1;
        d.mask_sum = clean_sum;
    } else {
        d.fallback = 1;
        d.mask_sum = base_sum;
    }
    d.candidate = d.mask_sum <= 0.0f ? 0 : 1;
    return d;
}

// startTime / endTime (:589-590): chunkOffsetSeconds + Double(frame) * frameDuration
FA_HD double frame_time(double chunk_offset, int frame, double frame_duration) {
    return d_add(chunk_offset, d_mul((double)frame, frame_duration));
}

// maskCosineSimilarity (:835-842) from the three dot products.
FA_HD float mask_cosine(float dot, float norm_a, float norm_b) {
    const float denom = f_mul(f_sqrt(norm_a), f_sqrt(norm_b));
    return denom > 0.0f ? f_div(dot, denom) : 0.0f;
}

// The order in which a mask CTA adds n values (vDSP_sve's own order is closed): lane t of kSumLanes adds v(t),
// v(t + kSumLanes), ... in turn from 0, then the lanes are folded in halves, lane t += lane t + h for h = 128 .. 1.
// The reference only ever sums binary weights, whose sums are exact integers in any order.
template <typename V> inline float ordered_sum(V v, int n) {
    float lane[kSumLanes];
    for (int t = 0; t < kSumLanes; ++t) {
        float a = 0.0f;
        for (int i = t; i < n; i += kSumLanes) a = f_add(a, v(i));
        lane[t] = a;
    }
    for (int h = kSumLanes / 2; h > 0; h >>= 1)
        for (int t = 0; t < h; ++t) lane[t] = f_add(lane[t], lane[t + h]);
    return lane[0];
}

} // namespace prepare
} // namespace fa
