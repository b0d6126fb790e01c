// Arithmetic of streaming speaker tracking (online_diar_kernels.cu), host and device: DiarizerManager's chunk logic
// around the pyannote segmentation and WeSpeaker embedding models, and SpeakerManager's assignment into a per-session
// speaker database.  Plain C++ on the host, so the CPU test-suite compiles it with g++ (tests/emul/online_diar_emul.cpp)
// and the C ABI runs the database operations on a host copy of one session with the same functions.
//
// The reference reduces 256-long vectors with closed vDSP code (vDSP_dotpr, vDSP_svesq).  Here every such reduction
// has one order, tree_sum: lane l (0..31) folds elements l, l + 32, ..., l + 224 left to right, then the 32 lane sums
// meet in an xor butterfly at distances 16, 8, 4, 2, 1.  A warp computes exactly that with __shfl_xor_sync, and every
// add and multiply is individually rounded (fa_float.cuh), so the kernel, this host build and the oracle agree bit for
// bit.  The left folds the Swift source spells out (validateEmbedding's map-reduce, the raw-embedding mean, the
// activity sums) stay left folds.
#pragma once

#include "../fa_common.cuh"
#include "../fa_float.cuh"

#include <cmath>
#include <cstdint>

namespace fa {
namespace od {

using namespace fa::fp;

constexpr int kDim = 256;                 // SpeakerManager.embeddingSize
constexpr int kFifo = 50;                 // Speaker.addRawEmbedding's FIFO depth
constexpr int kClasses = 7;               // powerset classes of the segmentation model
constexpr int kLocal = 3;                 // local speakers per chunk
constexpr int kModelSamples = 160000;     // the segmentation and embedding models' waveform length
constexpr double kFrameStep = 0.016875;   // SlidingWindow.step, seconds per frame
constexpr float kAlpha = 0.9f;            // updateMainEmbedding's EMA weight
constexpr float kEps = 1e-12f;            // VDSPOperations.l2Normalize's epsilon
constexpr float kUnitTolerance = 1e-3f;   // SpeakerUtilities.normalizationTolerance

// The powerset classes' speaker bits: [], [0], [1], [2], [0, 1], [0, 2], [1, 2]
FA_HD int class_bits(int c) {
    return c == 0 ? 0 : c <= 3 ? 1 << (c - 1) : c == 4 ? 3 : c == 5 ? 5 : 6;
}

// vDSP_maxvi over one frame's 7 logits: the first index of the maximum.  The running maximum starts at logit 0 and
// moves only on a strictly greater logit, so a NaN is never chosen past index 0, and a NaN at index 0 keeps index 0.
FA_HD int powerset_argmax(const float *x) {
    int best = 0;
    float m = x[0];
    for (int c = 1; c < kClasses; ++c)
        if (x[c] > m) {
            m = x[c];
            best = c;
        }
    return best;
}

// A frame's clean-frame mask for local speaker s: binarized and at most one speaker active (speaker sum < 2)
FA_HD int clean_mask(int bits, int s) {
    const int n = (bits & 1) + ((bits >> 1) & 1) + ((bits >> 2) & 1);
    return ((bits >> s) & 1) && n < 2;
}

// EmbeddingExtractor's numMasksInChunk for `samples` audio samples and F frames
FA_HD long long masks_in_chunk(long long frames, long long samples) {
    const long long n = (frames * samples + 80000) / 160000;
    return n < frames ? n : frames;
}

// ---- the pinned 256-long reductions
struct Lanes {
    float v[32];
};

FA_HD float butterfly(Lanes p) {
    for (int o = 16; o >= 1; o >>= 1) {
        Lanes q;
        for (int l = 0; l < 32; ++l) q.v[l] = f_add(p.v[l], p.v[l ^ o]);
        p = q;
    }
    return p.v[0];
}

FA_HD float tree_dot(const float *a, const float *b) {
    Lanes p;
    for (int l = 0; l < 32; ++l) {
        float s = f_mul(a[l], b[l]);
        for (int k = 1; k < 8; ++k) s = f_add(s, f_mul(a[l + 32 * k], b[l + 32 * k]));
        p.v[l] = s;
    }
    return butterfly(p);
}

// VDSPOperations.l2Normalize: x * (1 / max(sqrt(x . x), 1e-12)), from the sum of squares `ss`
FA_HD float norm_scale(float ss) { return f_div(1.0f, swift_max(f_sqrt(ss), kEps)); }

FA_HD void l2_normalize(const float *x, float *y) {
    const float scale = norm_scale(tree_dot(x, x));
    for (int i = 0; i < kDim; ++i) y[i] = f_mul(x[i], scale);
}

// SpeakerUtilities.cosineDistance from the dot product and the two sums of squares
FA_HD float cosine_from(float dot, float ssa, float ssb) {
    if (!(ssa > 0.0f && ssb > 0.0f)) return INFINITY;
    float sim;
    if (fabsf(f_sub(ssa, 1.0f)) <= kUnitTolerance && fabsf(f_sub(ssb, 1.0f)) <= kUnitTolerance) {
        sim = dot;
    } else {
        const float ma = f_sqrt(ssa), mb = f_sqrt(ssb);
        if (!(ma > 0.0f && mb > 0.0f)) return INFINITY;
        sim = f_div(dot, f_mul(ma, mb));
    }
    return f_sub(1.0f, swift_min(swift_max(sim, -1.0f), 1.0f));
}

FA_HD float cosine_distance(const float *a, const float *b) {
    return cosine_from(tree_dot(a, b), tree_dot(a, a), tree_dot(b, b));
}

// AudioValidation.validateEmbedding: every element finite, and sqrt of the left fold of squares above 0.1
FA_HD bool valid_embedding(const float *e) {
    float ss = 0.0f;
    for (int i = 0; i < kDim; ++i) {
        if (!(fabsf(e[i]) < INFINITY)) return false;   // NaN or infinite
        ss = f_add(ss, f_mul(e[i], e[i]));
    }
    return f_sqrt(ss) > 0.1f;
}

// calculateEmbeddingQuality: min(1, sqrt(vDSP.sumOfSquares(e)) / 10)
FA_HD float embedding_quality(const float *e) { return swift_min(1.0f, f_div(f_sqrt(tree_dot(e, e)), 10.0f)); }

// updateMainEmbedding's EMA step for one dimension, before its normalisation
FA_HD float ema(float current, float fresh) {
    return f_add(f_mul(kAlpha, current), f_mul(f_sub(1.0f, kAlpha), fresh));
}

// ---- thresholds a config resolves to (DiarizerManager.init, DiarizerConfig)
struct Resolved {
    float speaker_threshold;     // clusteringThreshold * 1.2
    float embedding_threshold;   // clusteringThreshold * 0.8
    float min_speech;            // minSpeechDuration: new speakers and segments
    float min_active;            // minActiveFramesCount
};

// ---- one speaker of a session's database, as it lies in HBM
struct SpeakerMeta {
    long long key;            // identity: the value of a canonical decimal id (named == 0), else the caller's key
    long long numeric;        // Int(id) when has_numeric
    long long update_count;
    long long raw_seq[kFifo]; // per-handle sequence numbers of the raw embeddings (their timestamps)
    float duration;
    int named, has_numeric, permanent;
    int raw_count, raw_head;  // the FIFO of raw embeddings: raw_count rows from ring index raw_head
};

struct Speaker {
    float current[kDim];
    float raw[kFifo][kDim];
    SpeakerMeta m;
};

// Per-session database header
struct SessionMeta {
    long long count;     // speakers, in insertion order
    long long next_id;   // nextSpeakerId
};

FA_HD const float *raw_row(const Speaker &s, int j) { return s.raw[(s.m.raw_head + j) % kFifo]; }

// Speaker.recalculateMainEmbedding: the mean of the raws in FIFO order, normalised
FA_HD void recalculate(Speaker &s) {
    if (s.m.raw_count == 0) return;
    float avg[kDim];
    for (int i = 0; i < kDim; ++i) {
        float a = 0.0f;
        for (int j = 0; j < s.m.raw_count; ++j) a = f_add(a, raw_row(s, j)[i]);
        avg[i] = f_div(a, (float)s.m.raw_count);
    }
    l2_normalize(avg, s.current);
}

// Speaker.addRawEmbedding of an already normalised row (RawEmbedding.init normalises its input; `row` is that result)
FA_HD void add_raw(Speaker &s, const float *row, long long seq) {
    if (!(tree_dot(row, row) > 0.01f)) return;
    if (s.m.raw_count >= kFifo) {
        s.m.raw_head = (s.m.raw_head + 1) % kFifo;
        --s.m.raw_count;
    }
    const int at = (s.m.raw_head + s.m.raw_count) % kFifo;
    for (int i = 0; i < kDim; ++i) s.raw[at][i] = row[i];
    s.m.raw_seq[at] = seq;
    ++s.m.raw_count;
    recalculate(s);
}

// Speaker.updateMainEmbedding(duration:embedding:alpha: 0.9) of the assignment's normalised embedding `n`
FA_HD void update_main(Speaker &s, const float *n, float duration, long long seq) {
    if (!(tree_dot(n, n) > 0.01f)) return;
    float ne[kDim], raw[kDim];
    l2_normalize(n, ne);
    l2_normalize(ne, raw);
    add_raw(s, raw, seq);
    float c[kDim];
    for (int i = 0; i < kDim; ++i) c[i] = ema(s.current[i], ne[i]);
    l2_normalize(c, s.current);
    s.m.duration = f_add(s.m.duration, duration);
    ++s.m.update_count;
}

// createNewSpeaker's record for id `id` from the assignment's normalised embedding `n`: normalised again on the way
// in, by Speaker.init and by RawEmbedding.init
FA_HD void new_speaker(Speaker &s, const float *n, float duration, long long id, long long seq) {
    float ne[kDim], raw[kDim];
    l2_normalize(n, ne);
    l2_normalize(ne, s.current);
    s.m = SpeakerMeta{};
    s.m.key = id;
    s.m.numeric = id;
    s.m.has_numeric = 1;
    s.m.update_count = 1;
    s.m.duration = duration;
    l2_normalize(ne, raw);
    add_raw(s, raw, seq);
}

// The index of the speaker with canonical id `id`, or -1
FA_HD long long find_canonical(const Speaker *db, long long count, long long id) {
    for (long long i = 0; i < count; ++i)
        if (!db[i].m.named && db[i].m.key == id) return i;
    return -1;
}

// findClosestSpeaker in insertion order: the first speaker at the least distance below +inf (a NaN never matches).
// Returns its index, or -1 with *distance = +inf.
FA_HD long long closest(const Speaker *db, long long count, const float *q, float *distance) {
    long long best = -1;
    float m = INFINITY;
    for (long long i = 0; i < count; ++i) {
        const float d = cosine_distance(q, db[i].current);
        if (d < m) {
            m = d;
            best = i;
        }
    }
    *distance = m;
    return best;
}

// SpeakerManager.assignSpeaker of one raw embedding `e` (its duration already formed); db has room for one more.
// Returns the index of the speaker it went to, or -1 when the segment is too short for a new speaker.
FA_HD long long assign_speaker(Speaker *db, SessionMeta &meta, const float *e, float duration, const Resolved &r,
                               long long seq) {
    float n[kDim], d;
    l2_normalize(e, n);
    const long long i = closest(db, meta.count, n, &d);
    if (i >= 0 && d < r.speaker_threshold) {
        if (d < r.embedding_threshold) update_main(db[i], n, duration, seq);
        else db[i].m.duration = f_add(db[i].m.duration, duration);
        return i;
    }
    if (!(duration >= r.min_speech)) return -1;
    const long long id = meta.next_id++;
    long long at = find_canonical(db, meta.count, id);   // speakerDatabase[newSpeakerId] = ...: an old id is replaced
    if (at < 0) at = meta.count++;
    new_speaker(db[at], n, duration, id, seq);
    return at;
}

// One chunk's assignment (DiarizerManager.swift:351-378): local speakers strictly in order.  activity[s]: the
// binarized column sum; need bit s: the embedding model ran for s (else its embedding is zero).  assigned[s]: the
// speaker's index, or -1 (no id).  db has room for three more speakers.
FA_HD void assign_chunk(Speaker *db, SessionMeta &meta, const float *emb, const float *activity, int need,
                        const Resolved &r, long long seq0, long long *assigned) {
    for (int s = 0; s < kLocal; ++s) {
        assigned[s] = -1;
        if (!(activity[s] > r.min_active) || !((need >> s) & 1) || !valid_embedding(emb + s * kDim)) continue;
        const float duration = f_mul(activity[s], (float)kFrameStep);
        assigned[s] = assign_speaker(db, meta, emb + s * kDim, duration, r, seq0 + s);
    }
}

// ---- segments (createTimedSegments / createSegmentIfValid)
struct Segment {
    int speaker;             // local speaker 0..2
    float start, end, quality;
};

// Most segments one chunk of F frames yields: runs of one speaker are separated by an inactive frame
FA_HD long long segment_bound(long long frames) { return kLocal * ((frames + 1) / 2); }

// Segments of one chunk from its binarized frames (bit s of bits[f]: local speaker s), sorted by start time.  Swift's
// sort is not stable; equal start times keep the order the segments are made in (local speaker 0, 1, 2).
// has_id[s]: the speaker got an id; quality[s]: its embedding's quality.  `made` and `out` hold
// segment_bound(frames) each; returns the count.
FA_HD int chunk_segments(const unsigned char *bits, int frames, const float *activity, const int *has_id,
                         const float *quality, double offset, const Resolved &r, Segment *made, Segment *out) {
    int n = 0;
    int first[kLocal + 1];
    Segment *const keep = out;
    out = made;
    for (int s = 0; s < kLocal; ++s) {
        first[s] = n;
        if (activity[s] < r.min_active || !has_id[s]) continue;
        bool active = false;
        int start = 0;
        for (int f = 0; f <= frames; ++f) {
            bool on = false;
            if (f < frames) {   // the dynamic threshold: 0.15 while another speaker is above 0.3, else 0.3
                const float x = (float)((bits[f] >> s) & 1);
                float th = 0.3f;
                for (int o = 0; o < kLocal; ++o)
                    if (o != s && (float)((bits[f] >> o) & 1) > 0.3f) {
                        th = 0.15f;
                        break;
                    }
                on = x > th;
            }
            if (on && !active) {
                active = true;
                start = f;
            } else if (!on && active) {
                const double t0 = offset + (double)start * kFrameStep, t1 = offset + (double)f * kFrameStep;
                if (!((float)(t1 - t0) < r.min_speech))
                    out[n++] = Segment{s, (float)t0, (float)t1,
                                       f_mul(quality[s], f_div(activity[s], (float)(f - start)))};
                active = false;
            }
        }
    }
    first[kLocal] = n;
    // stable merge of the three lists, each already in start order (a run starts after its speaker's previous run)
    int at[kLocal] = {first[0], first[1], first[2]};
    for (int k = 0; k < n; ++k) {
        int pick = -1;
        for (int s = 0; s < kLocal; ++s)
            if (at[s] < first[s + 1] && (pick < 0 || made[at[s]].start < made[at[pick]].start)) pick = s;
        keep[k] = made[at[pick]++];
    }
    return n;
}

} // namespace od
} // namespace fa
