// Arithmetic of voice activity detection (vad_kernels.cu), host and device: the Silero chunk staging, the streaming
// hysteresis, speech segmentation with O(1) state per clip, and the FSMN-VAD decision.  Plain C++ on the host, so the
// CPU test-suite compiles it with g++ (tests/emul/vad_emul.cpp).
#pragma once

#include "../fa_common.cuh"

#include <cstdint>

namespace fa {
namespace vad {

constexpr int kChunk = 4096;                       // VadManager.chunkSize
constexpr int kContext = 64;                       // VadState.contextLength
constexpr int kState = 128;                        // VadManager.stateSize
constexpr int kModelInput = kContext + kChunk;     // VadManager.modelInputSize, 4160
constexpr long long kNil = -1;                     // tempEndSample == nil; sample positions are never negative

struct Resolved {
    float threshold, negative, split;
    int use_max;
    long long min_speech, min_silence, max_speech, pad, min_silence_at_max;
};

// Swift's global min and max (y < x ? y : x and y >= x ? y : x): a NaN argument is kept or dropped by position
FA_HD float swift_min(float x, float y) { return y < x ? y : x; }
FA_HD float swift_max(float x, float y) { return y >= x ? y : x; }
FA_HD long long lmax(long long a, long long b) { return a > b ? a : b; }
FA_HD long long lmin(long long a, long long b) { return a < b ? a : b; }

// Sample j (0 .. 4095) of the processed chunk (VadManager.processChunk, :171-182): truncation to the first 4096
// samples, or repeat-last padding (0 for an empty chunk)
FA_HD float chunk_sample(const float *x, long long n, int j) {
    return j < n ? x[j] : (n > 0 ? x[n - 1] : 0.0f);
}

// ---- streamingStateMachine (VadManager+Streaming.swift:31-91)
struct StreamState {
    long long processed, temp_end;   // processedSamples, tempEndSample (kNil)
    long long triggered;
};

enum : int { kEventNone = 0, kEventStart = 1, kEventEnd = 2 };

// One committed chunk of n samples with probability p; returns the event kind and its sample in *sample (-1: none)
FA_HD int stream_step(StreamState &s, float p, long long n, const Resolved &r, long long *sample) {
    *sample = -1;
    s.processed += n;
    if (p >= r.threshold) {
        s.temp_end = kNil;
        if (!s.triggered) {
            s.triggered = 1;
            *sample = lmax(0, s.processed - r.pad - n);
            return kEventStart;
        }
    } else if (p < r.negative && s.triggered) {
        if (s.temp_end == kNil) s.temp_end = s.processed;
        if (s.processed - s.temp_end >= r.min_silence) {
            *sample = lmax(0, s.temp_end + r.pad - n);
            s.triggered = 0;
            s.temp_end = kNil;
            return kEventEnd;
        }
    }
    return kEventNone;
}

// ---- detectSpeechSampleRanges (VadManager+SpeechSegmentation.swift:71-234) in O(1) state.
// The split choice reads three entries of possibleEnds: the first longest candidate whose minProbability <= split
// (Sequence.max(by:) keeps the first of equal maxima), the first longest overall, and the last.  Each is kept as the
// candidates arrive.  The padding pass (:205-224) changes a range's end and the next range's start only, so it runs
// one raw range behind, and the final clamp and filter (:226-233) go with it.  Segments go to out[2k], out[2k + 1].
struct Candidate {
    long long start, duration;
};

struct Segmenter {
    const Resolved &r;
    long long L;            // audioLengthSamples
    long long *out;
    long long n = 0;        // segments written
    bool has_pend = false;
    long long pend_s = 0, pend_e = 0;
    long long cur = 0;      // currentSpeechStart

    FA_HD Segmenter(const Resolved &res, long long length, long long *o) : r(res), L(length), out(o) {}

    FA_HD void emit(long long s, long long e) {
        const long long a = lmax(0, lmin(s, L)), b = lmax(a, lmin(e, L));
        if (b > a) {
            out[2 * n] = a;
            out[2 * n + 1] = b;
            ++n;
        }
    }
    FA_HD void raw(long long s, long long e) {
        if (!has_pend) {
            pend_s = lmax(0, s - r.pad);
            pend_e = e;
            has_pend = true;
            return;
        }
        const long long silence = s - pend_e;
        const long long step = silence < 2 * r.pad ? silence / 2 : r.pad;   // C++ and Swift both truncate toward 0
        pend_e = lmin(L, pend_e + step);
        emit(pend_s, pend_e);
        pend_s = lmax(0, s - step);
        pend_e = e;
    }
    FA_HD void flush(long long end) {   // flushCurrentSpeechEnd (:109-115)
        if (end <= cur) return;
        if (end - cur >= r.min_speech) raw(cur, lmin(end, L));
    }
    FA_HD void finish() {
        if (has_pend) emit(pend_s, lmin(L, pend_e + r.pad));
    }
};

// Segments of one clip of P chunk probabilities and L samples into out (at most P pairs); returns their count
FA_HD long long segment_clip(const float *p, long long P, long long L, const Resolved &r, long long *out) {
    if (P <= 0 || L <= 0) return 0;
    Segmenter g(r, L, out);
    bool triggered = false, has_min = false, has_below = false, has_any = false;
    long long temp_end = kNil;
    float temp_min = 0.0f;
    Candidate below{0, 0}, longest{0, 0}, last{0, 0};
    const bool bounded = r.max_speech < INT64_MAX;
    for (long long i = 0; i < P; ++i) {
        const long long fs = i * kChunk;
        const float prob = p[i];
        if (prob >= r.threshold) {
            if (temp_end != kNil) {
                const long long dur = fs - temp_end;
                if (dur > r.min_silence_at_max) {
                    const Candidate c{temp_end, dur};
                    const float mp = has_min ? temp_min : 1.0f;
                    if (mp <= r.split && (!has_below || dur > below.duration)) below = c, has_below = true;
                    if (!has_any || dur > longest.duration) longest = c;
                    last = c;
                    has_any = true;
                }
            }
            temp_end = kNil;
            has_min = false;
            if (!triggered) {
                triggered = true;
                g.cur = fs;
                continue;
            }
        }
        if (triggered && bounded && fs - g.cur > r.max_speech) {
            const bool chosen = has_any;
            const Candidate c = has_below ? below : (r.use_max ? longest : last);
            g.flush(chosen ? c.start : fs);
            if (chosen && c.start + c.duration < fs) {
                g.cur = c.start + c.duration;
            } else {
                triggered = false;
            }
            has_below = has_any = false;
            temp_end = kNil;
            has_min = false;
            if (!triggered) continue;
        }
        if (prob < r.negative && triggered) {
            if (temp_end == kNil) temp_end = fs;
            temp_min = swift_min(has_min ? temp_min : prob, prob);
            has_min = true;
            if (fs - temp_end >= r.min_silence) {
                g.flush(temp_end);
                triggered = false;
                temp_end = kNil;
                has_min = false;
                has_below = has_any = false;
                continue;
            }
        }
    }
    if (triggered) g.flush(L);
    g.finish();
    return g.n;
}

// ---- FsmnVadManager.decide(silence:) (FsmnVadManager.swift:159-201), its constants fixed (:37-45).  The 20-frame
// window is a bit mask.  A segment opens on one frame and closes on a later one (or at T), so a clip of T frames has at
// most (T + 1) / 2 segments.
constexpr float kFsmnSilence = 0.2f;
constexpr int kFsmnWindow = 20, kFsmnSilToSpeech = 15, kFsmnSpeechToSil = 15, kFsmnMaxEndSilence = 80,
              kFsmnLookback = 20, kFsmnLookahead = 10, kFsmnMaxSegment = 6000, kFsmnFrameMs = 10;

FA_HD long long fsmn_bound(long long T) { return (T + 1) / 2; }

FA_HD long long fsmn_clip(const float *sil, long long T, long long *out) {
    unsigned win = 0;
    int pos = 0, sum = 0, cont = 0;
    bool pre = false, in = false;
    long long start = 0, n = 0;
    for (long long t = 0; t < T; ++t) {
        const int cur = sil[t] <= kFsmnSilence ? 1 : 0;
        sum += cur - (int)((win >> pos) & 1u);
        win = (win & ~(1u << pos)) | ((unsigned)cur << pos);
        pos = pos + 1 == kFsmnWindow ? 0 : pos + 1;
        if (!pre && sum >= kFsmnSilToSpeech) {
            pre = true;
            if (!in) {
                in = true;
                start = lmax(0, t - kFsmnSilToSpeech - kFsmnLookback);
                cont = 0;
            }
        } else if (pre && sum <= kFsmnSpeechToSil) {
            pre = false;
        }
        cont = in && !pre ? cont + 1 : 0;
        if (in && cont >= kFsmnMaxEndSilence) {
            out[2 * n] = start * kFsmnFrameMs;
            out[2 * n + 1] = (t - kFsmnMaxEndSilence + kFsmnLookahead) * kFsmnFrameMs;
            ++n;
            in = false;
        } else if (in && t - start >= kFsmnMaxSegment) {
            out[2 * n] = start * kFsmnFrameMs;
            out[2 * n + 1] = t * kFsmnFrameMs;
            ++n;
            in = false;
            pre = false;
        }
    }
    if (in) {
        out[2 * n] = start * kFsmnFrameMs;
        out[2 * n + 1] = T * kFsmnFrameMs;
        ++n;
    }
    return n;
}

} // namespace vad
} // namespace fa
