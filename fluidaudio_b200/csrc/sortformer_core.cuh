// Per-element arithmetic of Sortformer's streaming state update (sortformer_kernels.cu), host- and device-callable so
// that the CPU suite runs the very code the kernels run (tests/emul/sortformer_emul.cpp).
//
// Reference (paths under Sources/FluidAudio/Diarizer/Sortformer):
//   SortformerTypes.swift:31-97,239-254        configuration and the init's clamps
//   SortformerStateUpdater.swift:31-165        streamingUpdate: lengths, FIFO, pop, first spkcachePreds
//   SortformerStateUpdater.swift:175-212       updateSilenceProfile
//   SortformerStateUpdater.swift:220-305       compressSpkcache
//   SortformerStateUpdater.swift:311-348       getLogPredScores
//   SortformerStateUpdater.swift:351-390       disableLowScores
//   SortformerStateUpdater.swift:393-457       boostTopKScores
//   SortformerStateUpdater.swift:465-578       getTopKIndices
//
// Every float32 operation the reference states is one round-to-nearest operation here (__f*_rn on the device, plain
// operators on the host, whose build keeps contraction off).  vForce.log / log1p are Accelerate's and closed: both
// sides compute the correctly rounded float32 log and log1p instead (fa_float.cuh, DESIGN §4.7).
//
// Both selections (the per-speaker boosts and the global top-k) are insertion sorts in the reference.  Each keeps the
// first k elements of a strict total order on (value, index) for non-NaN input, so an element is kept exactly when
// fewer than k elements precede it: `precedes` below is that order, and the kernels count ranks with it.
#pragma once

#include "fa_common.cuh"
#include "fa_float.cuh"

#include <cmath>

namespace fa {
namespace sortformer {

constexpr int kSpeakers = 4;     // numSpeakers (let)
constexpr int kDims = 512;       // preEncoderDims (let)
constexpr int kMaxIndex = 99999; // maxIndex (let)
constexpr float kLn2 = 0.693147182f;   // logf(2) = -logf(0.5), correctly rounded

using namespace fa::fp;   // f_add / f_sub / f_mul / f_div / f_log / f_log1p (fa_float.cuh)

// Resolved configuration: the fields of fa_sortformer_config after the init's clamps, plus the derived top-k sizes.
struct Config {
    int chunk_len, left_context, right_context, fifo_len, spkcache_len, update_period, sil_per_spk;
    float silence_threshold, pred_score_threshold, scores_boost_latest, strong_boost_rate, weak_boost_rate,
        min_pos_scores_rate;
    int max_core;                         // the largest coreFrames a push may carry
    int strong_k, weak_k, min_pos;        // compressSpkcache (:229-232)
    FA_HD int fifo_rows() const { return fifo_len + max_core; }                    // FIFO ring capacity
    FA_HD int cache_rows() const { return spkcache_len + fifo_len + max_core; }    // speaker cache before compression
};

// Int(Float(perSpk) * rate) (:230-232); Swift traps outside Int's range, rates are checked finite at create
FA_HD int scaled_count(int per_spk, float rate) {
    const float v = f_mul((float)per_spk, rate);
    return v >= 2147483520.0f ? 2147483520 : v <= -2147483520.0f ? -2147483520 : (int)v;
}

// vDSP.clip(x, lo...hi)
FA_HD float clip(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }

// getLogPredScores (:311-348) for one frame: p[4] -> s[4]
FA_HD void frame_scores(const float *p, float thr, float *s) {
    float l[kSpeakers];
    const float hi = f_sub(1.0f, thr);
    float sum = 0.0f;
    for (int k = 0; k < kSpeakers; ++k) {
        l[k] = f_log1p(-clip(p[k], 0.0f, hi));
        sum = f_add(sum, l[k]);
    }
    for (int k = 0; k < kSpeakers; ++k) {
        const float lp = f_log(clip(p[k], thr, 3.40282347e38f));
        s[k] = f_add(f_add(kLn2, f_sub(lp, l[k])), sum);
    }
}

// disableLowScores (:365): the positive-score count of the pre-disable scores
FA_HD bool positive_score(float p, float s) { return p > 0.5f && s > 0.0f; }

// disableLowScores (:371-387) and the latest-frame boost (:246-252) for one (frame, speaker)
FA_HD float disable_and_boost(float p, float s, int pos_count, int min_pos, bool latest, float boost_latest) {
    if (p <= 0.5f) s = -INFINITY;
    else if (s <= 0.0f && pos_count >= min_pos) s = -INFINITY;
    return latest ? f_add(s, boost_latest) : s;
}

// The order both selections keep: value descending, ties to the smaller index.
FA_HD bool precedes(float va, int ia, float vb, int ib) { return va > vb || (va == vb && ia < ib); }

// How many of the n elements (at(j), j) precede (v, i), counting stops at k: the element is kept when the result is
// below k.  The per-speaker boosts skip -inf elements (:419); the global selection counts them (:494-541).
template <typename At> FA_HD int rank_until(At at, int n, float v, int i, int k, bool skip_neg_inf) {
    int rank = 0;
    for (int j = 0; j < n && rank < k; ++j) {
        const float w = at(j);
        rank += (!(skip_neg_inf && w == -INFINITY) && precedes(w, j, v, i)) ? 1 : 0;
    }
    return rank;
}

// boostTopKScores (:393-457): boost of a kept element; -inf is never kept
FA_HD float boost(float v, float scale) { return f_add(v, f_mul(scale, kLn2)); }

// updateSilenceProfile (:185-210): Σ_spk p in order, and one dimension's running-mean step
FA_HD float prob_sum(const float *p) {
    float s = 0.0f;
    for (int k = 0; k < kSpeakers; ++k) s = f_add(s, p[k]);
    return s;
}
FA_HD float mean_step(float old_mean, float x, float n) { return f_div(f_add(f_mul(old_mean, n), x), f_add(n, 1.0f)); }

// getTopKIndices (:543-577): a kept permuted index and its value -> the index before sorting (maxIndex for -inf)
FA_HD int kept_index(float v, int permuted) { return v == -INFINITY ? kMaxIndex : permuted; }

} // namespace sortformer
} // namespace fa
