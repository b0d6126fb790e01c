// Per-lane arithmetic of the diarizer timelines (timeline_kernels.cu): DiarizerTimeline's segment detection for one
// (session, speaker), host- and device-callable so that the CPU suite runs the very code the kernel runs
// (tests/emul/timeline_emul.cpp).
//
// Reference (Sources/FluidAudio/Diarizer/DiarizerTimeline.swift):
//   :9-164        DiarizerTimelineConfig
//   :602-619      DiarizerActivityType.evaluationFunction
//   :649-661      SegmentScratch
//   :827-872      _addChunkUnlocked: the finalized pass, whose scratch is kept, then the tentative pass on a copy
//   :1169-1294    updateSegments
//   :1297-1336    commitSegment
//
// Every float32 operation the reference states is one round-to-nearest operation (fa_float.cuh).  Frame indices are
// int64 (Swift's Int) and the `.min` sentinels are INT64_MIN; create rejects negative pads and minimum durations, which
// would overflow them (Swift traps there).  `.logits` is log(c / (1 - c)) with f_log the correctly rounded float32 log (DESIGN §4.8).
#pragma once

#include "../../include/fluidaudio_b200.h"
#include "fa_common.cuh"
#include "fa_float.cuh"

#include <cstdint>

namespace fa {
namespace timeline {

using namespace fa::fp;

constexpr int kMaxSpeakers = 32;   // one warp per session, one lane per speaker
constexpr long long kMinFrame = INT64_MIN;

enum : int { kSigmoids = 0, kLogits = 1 };

// The numeric fields of DiarizerTimelineConfig a pass reads.
struct Params {
    float onset, offset;
    int pad_on, pad_off, min_on, min_off;
    int activity;   // kSigmoids or kLogits
};

// SegmentScratch (:649-661).
struct Scratch {
    long long start, end, unmerged_start;
    long long count, unmerged_count;   // activeFrameCount, unmergedActiveFrameCount
    float sum, unmerged_sum;           // activitySum, unmergedActivitySum
    int speaking, has_segment;
};

// A segment as the C ABI returns it: {start_frame, end_frame, activity, speaker}.
using Segment = fa_diarizer_timeline_segment;

// A scratch in HBM stores its three frames XOR 2^63, so that all-zero bytes are a fresh scratch: open, reset and
// clearing one speaker are memsets.
struct StoredScratch {
    unsigned long long start, end, unmerged_start;
    long long count, unmerged_count;
    float sum, unmerged_sum;
    int speaking, has_segment;
};
constexpr unsigned long long kFrameBias = 0x8000000000000000ull;
FA_HD Scratch load_scratch(const StoredScratch &s) {
    return Scratch{(long long)(s.start ^ kFrameBias), (long long)(s.end ^ kFrameBias),
                   (long long)(s.unmerged_start ^ kFrameBias), s.count, s.unmerged_count, s.sum, s.unmerged_sum,
                   s.speaking, s.has_segment};
}
FA_HD StoredScratch store_scratch(const Scratch &s) {
    return StoredScratch{(unsigned long long)s.start ^ kFrameBias, (unsigned long long)s.end ^ kFrameBias,
                         (unsigned long long)s.unmerged_start ^ kFrameBias, s.count, s.unmerged_count, s.sum,
                         s.unmerged_sum, s.speaking, s.has_segment};
}

// evaluationFunction (:607-618)
FA_HD float activity_of(float p, int type) {
    if (type == kSigmoids) return p;
    const float eps = 1e-6f;
    const float c = swift_min(swift_max(p, eps), f_sub(1.0f, eps));
    return f_log(f_div(c, f_sub(1.0f, c)));
}

// The most segments one speaker emits in a push of n finalized and m tentative rows: ceil((n + m) / 2) + 1.
//
// Emissions are the onset commits, the end-of-pass commit of a held segment and the trailing tentative segment.  Onsets
// and closures alternate, an onset commits only after a closure (or a held segment carried in), and `speaking` implies
// no held segment, so the end-of-pass commit and the trailing one exclude each other.  Counting both passes over every
// entry state (speaking, holding a segment, neither) gives max(ceil(n/2) + floor(m/2), floor(n/2) + ceil(m/2)) + 1.
// For odd n and m it is the exact maximum: alternating 0/1 input reaches it from a speaking lane with the default
// thresholds (tests/test_diarizer_timeline.py).  The staging slot of each lane holds this many segments.
FA_HD long long segment_bound(long long n, long long m) { return (n + m + 1) / 2 + 1; }
// Of which finalized (only the finalized pass emits them) and tentative (only the tentative pass): each list's own bound.
FA_HD long long finalized_bound(long long n) { return n > 0 ? n / 2 + 1 : 0; }
FA_HD long long tentative_bound(long long m) { return (m + 1) / 2 + 1; }

// commitSegment (:1297-1336) without the speaker store, which the host façade keeps.
template <typename Emit> FA_HD void commit(Scratch &a, int spk, bool finalized, Emit &emit) {
    if (!a.has_segment) return;
    const float activity = a.count > 0 ? f_div(a.sum, (float)a.count) : 0.0f;
    emit(Segment{a.start, a.end, activity, spk}, finalized);
    a.has_segment = 0;
    a.sum = 0.0f;
    a.count = 0;
}

// updateSegments (:1169-1294) for speaker `spk`: rows row(i), i < n, are frames offset + i.  emit(segment, finalized)
// receives the segments in the order the reference appends them.
template <typename Row, typename Emit>
FA_HD void update_pass(const Params &c, Scratch &a, int spk, long long offset, long long n, Row &&row, bool finalized,
                       bool trailing, Emit &emit) {
    if (n == 0 && !trailing) return;   // guard !predictions.isEmpty || addTrailingTentative
    const long long end_frame = offset + n;
    const long long pad = (long long)c.pad_on + c.pad_off;
    const long long min_len = pad + c.min_on;
    const long long finalized_end = finalized ? end_frame - c.min_off - pad : kMinFrame;
    for (long long i = 0; i < n; ++i) {
        const float p = row(i);
        const long long frame = offset + i;
        if (a.speaking) {
            if (p >= c.offset) {
                a.unmerged_sum = f_add(a.unmerged_sum, activity_of(p, c.activity));
                a.unmerged_count += 1;
                continue;
            }
            a.speaking = 0;
            const long long end = frame + c.pad_off;
            if (!(end >= a.unmerged_start + min_len)) {
                a.has_segment = a.end >= a.start + min_len;
                continue;
            }
            a.end = end;
            a.sum = f_add(a.sum, a.unmerged_sum);
            a.count += a.unmerged_count;
            a.has_segment = 1;
        } else if (p > c.onset) {
            const long long start = frame - c.pad_on;
            a.speaking = 1;
            a.unmerged_start = start;
            a.unmerged_sum = activity_of(p, c.activity);
            a.unmerged_count = 1;
            if (!(!a.has_segment || start > a.end + c.min_off)) {
                a.has_segment = 0;
                continue;
            }
            commit(a, spk, finalized, emit);
            a.start = start;
        }
    }
    if (a.has_segment && (!finalized || a.end < finalized_end)) commit(a, spk, finalized && a.end < finalized_end, emit);
    if (finalized || !trailing || !a.speaking) return;
    const long long padded_end = end_frame + c.pad_off;
    if (!(padded_end >= a.start + min_len)) return;
    a.has_segment = 1;
    if (padded_end >= a.unmerged_start + min_len) {
        a.end = padded_end;
        a.sum = f_add(a.sum, a.unmerged_sum);
        a.count += a.unmerged_count;
    }
    commit(a, spk, false, emit);
}

// One push for one speaker (_addChunkUnlocked, :833-865): the finalized pass over n rows from the finalized cursor,
// whose scratch `a` keeps, then the tentative pass over m rows on a copy.
template <typename FinRow, typename TenRow, typename Emit>
FA_HD void push_lane(const Params &c, Scratch &a, int spk, long long cursor, long long n, FinRow &&fin, long long m,
                     TenRow &&ten, Emit &emit) {
    update_pass(c, a, spk, cursor, n, fin, true, false, emit);
    Scratch t = a;
    update_pass(c, t, spk, cursor + n, m, ten, false, true, emit);
}

} // namespace timeline
} // namespace fa
