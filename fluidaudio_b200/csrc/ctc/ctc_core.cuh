// Host- and device-callable arithmetic of CTC keyword spotting (ctc_kernels.cu; its host build is tests/emul/
// ctc_emul.cpp): CtcKeywordSpotter.applyLogSoftmax / makeLogProbs (CtcKeywordSpotter.swift:268-306,
// CtcKeywordSpotter+Inference.swift:350-431), mergeOverlapFrame (+Inference.swift:329-346) and the CTC-WS dynamic
// program of CtcDPAlgorithm (CtcDPAlgorithm.swift:121-392), one cell, one frame's candidate test and one pair's merge
// at a time.  Every float operation is one fa::fp helper, so the kernels and the host build compute the same bits.
#pragma once

#include "../fa_float.cuh"

#include <cfloat>
#include <cstdint>

namespace fa {
namespace ctc {

constexpr int kWildcard = -1;        // ContextBiasingConstants.wildcardTokenId
constexpr int kStatesPerLane = 8;    // expanded states each lane of a pair's warp owns
constexpr int kMaxStates = 32 * kStatesPerLane;
constexpr int kMaxTokens = (kMaxStates - 1) / 2;   // 2N + 1 expanded states must fit one warp: N <= 127
constexpr int kBaselineTokens = 3;                  // ContextBiasingConstants.baselineTokenCountForThreshold
constexpr float kRelaxPerToken = 1.0f;              // ContextBiasingConstants.thresholdRelaxationPerToken
constexpr float kDefaultMinScore = -15.0f;          // ContextBiasingConstants.defaultMinSpotterScore
constexpr float kNeg = -FLT_MAX;                    // -Float.greatestFiniteMagnitude
constexpr float kLog2 = 0.69314718f;

// ------------------------------------------------------------------------------------------------ log-softmax
// One row of applyLogSoftmax: x(v) reads logit v, out(v, value) writes log-prob v.  Temperature division only when it
// is not 1, the max as Sequence.max() finds it (a later element replaces the running max only when it is greater), the
// exp sum in index order, then (x - max) - log(sum) and the blank bias when it is non-zero and blank_id < V.
template <typename In, typename Out>
FA_HD void log_softmax_row(int V, float temperature, float blank_bias, int blank_id, In x, Out out) {
    using namespace fp;
    const bool scale = temperature != 1.0f;
    auto scaled = [&](int v) { return scale ? f_div(x(v), temperature) : x(v); };
    float m = scaled(0);
    for (int v = 1; v < V; ++v) {
        const float e = scaled(v);
        if (m < e) m = e;
    }
    float sum = 0.0f;
    for (int v = 0; v < V; ++v) sum = f_add(sum, f_exp(f_sub(scaled(v), m)));
    const float lse = f_log(sum);
    const bool bias = blank_bias != 0.0f && blank_id < V;
    for (int v = 0; v < V; ++v) {
        const float r = f_sub(f_sub(scaled(v), m), lse);
        out(v, bias && v == blank_id ? f_sub(r, blank_bias) : r);
    }
}

// mergeOverlapFrame for one column: (m + log(exp(a - m) + exp(b - m))) - log 2 with m = Swift.max(a, b), -inf when m is.
FA_HD float merge_overlap(float a, float b) {
    using namespace fp;
    const float m = swift_max(a, b);
    if (m == -INFINITY) return -INFINITY;
    return f_sub(f_add(m, f_log(f_add(f_exp(f_sub(a, m)), f_exp(f_sub(b, m))))), kLog2);
}

// ------------------------------------------------------------------------------------------------ the expanded graph
// How state s of [B, t1, B, ..., tN, B] emits: a column of the frame, 0 or -FLT_MAX.
enum : int { kEmitZero = -1, kEmitNeg = -2 };
struct State {
    int col;         // column read, or kEmitZero / kEmitNeg
    bool match;      // a token or wildcard state: its last-token frame is the current frame
    bool can_skip;   // canSkipBlank: s - 2 may advance straight into s
};

// State s (0 .. 2N) of a term whose tokens tok(0 .. N-1) gives; V the vocabulary size.
template <typename Tok> FA_HD State expanded_state(int s, Tok tok, int V, int blank_id) {
    if ((s & 1) == 0) return State{blank_id >= 0 && blank_id < V ? blank_id : kEmitZero, false, false};
    const int id = tok(s >> 1);
    State st;
    st.match = true;
    if (id == kWildcard) {
        st.col = kEmitZero;
        st.can_skip = s < 2 || tok((s >> 1) - 1) != kWildcard;
    } else {
        st.col = id >= 0 && id < V ? id : kEmitNeg;
        st.can_skip = s < 2 || tok((s >> 1) - 1) != id;
    }
    st.can_skip = st.can_skip && s >= 2;
    return st;
}

FA_HD float emission(const State &st, const float *row) {
    return st.col >= 0 ? row[st.col] : (st.col == kEmitZero ? 0.0f : kNeg);
}

// One cell: dpI / startI / lastTokI of state s at frame t from the three predecessors at t - 1 (stay s, advance s - 1,
// skip s - 2; `skip` is ignored when the state cannot skip).  Ties prefer stay over advance over skip; a cell whose best
// predecessor is at or below -FLT_MAX / 2 is -FLT_MAX with start and last-token 0.
struct Cell {
    float dp;
    int start, last;
};
FA_HD Cell step_cell(const Cell &stay, const Cell &adv, const Cell &skip, const State &st, float added, int t, int s) {
    float best = stay.dp;
    int kind = 0;
    if (adv.dp > best) {
        best = adv.dp;
        kind = 1;
    }
    const float sk = st.can_skip ? skip.dp : kNeg;
    if (sk > best) {
        best = sk;
        kind = 2;
    }
    if (best <= kNeg / 2) return Cell{kNeg, 0, 0};
    const int start = kind == 0 ? stay.start : (kind == 1 ? adv.start : skip.start);
    const int last = kind == 0 ? stay.last : (kind == 1 ? adv.last : skip.last);
    return Cell{fp::f_add(best, added), kind == 1 && s == 1 ? t - 1 : start, st.match ? t : last};
}

// dp[t][N] of the public view: the token state 2N - 1 unless the blank after it is strictly better.
FA_HD Cell project(const Cell &tok, const Cell &blank) { return tok.dp >= blank.dp ? tok : blank; }

// ------------------------------------------------------------------------------------------------ candidates
struct Candidate {
    float score;
    int start, end;
};

// The threshold spotKeywordsFromLogProbs gives a term of n tokens: base - max(0, n - 3) * 1.0, or -15 without a base.
FA_HD float term_threshold(bool has_base, float base, int n) {
    if (!has_base) return kDefaultMinScore;
    const int extra = n - kBaselineTokens > 0 ? n - kBaselineTokens : 0;
    return fp::f_sub(base, fp::f_mul((float)extra, kRelaxPerToken));
}

// ctcWordSpotMultiple's scan over t = N .. T, fed one frame at a time (push) and closed by finish: each frame is tested
// as a local maximum (>= the previous normalised value, > the next; -FLT_MAX past either end) once the next is known,
// and the first strict maximum is kept for the fallback.  emit(Candidate) receives the candidates in t order.
struct Scan {
    float norm;        // normalisation factor (non-wildcard count, 1 when 0)
    float min_score;
    float prev;        // normalised value of frame t - 2 (-FLT_MAX when it is before N)
    Candidate held;    // frame t - 1, waiting for its next value
    bool has_held;
    Candidate fallback;
    bool any;

    FA_HD void init(float norm_, float min_score_) {
        norm = norm_;
        min_score = min_score_;
        prev = kNeg;
        has_held = false;
        fallback = Candidate{kNeg, 0, 0};
        any = false;
    }
    template <typename Emit> FA_HD void test(float next, Emit &&emit) {
        if (held.score >= prev && held.score > next && held.score >= min_score) {
            emit(held);
            any = true;
        }
        prev = held.score;
    }
    template <typename Emit> FA_HD void push(const Cell &c, Emit &&emit) {
        const Candidate cur{fp::f_div(c.dp, norm), c.start, c.last};
        if (has_held) test(cur.score, emit);
        held = cur;
        has_held = true;
        if (cur.score > fallback.score) fallback = cur;
    }
    template <typename Emit> FA_HD void finish(Emit &&emit) {
        if (has_held) test(kNeg, emit);
        if (!any && fallback.score >= min_score) emit(fallback);
    }
};

// Stable sort of c[0 .. n) by start frame (insertion sort: the candidates of a scan arrive nearly sorted), then the
// reference's merge in place: a candidate that starts at or before the last merged end joins it, the higher score
// (ties keep the earlier) taking the max of both ends.  Returns the merged count.
FA_HD int merge_candidates(Candidate *c, int n) {
    for (int i = 1; i < n; ++i) {
        const Candidate x = c[i];
        int j = i;
        while (j > 0 && c[j - 1].start > x.start) {
            c[j] = c[j - 1];
            --j;
        }
        c[j] = x;
    }
    int m = 0;
    for (int i = 0; i < n; ++i) {
        if (m > 0 && c[i].start <= c[m - 1].end) {
            const Candidate last = c[m - 1];
            Candidate best = c[i].score > last.score ? c[i] : last;
            best.end = last.end >= c[i].end ? last.end : c[i].end;
            c[m - 1] = best;
        } else {
            c[m++] = c[i];
        }
    }
    return m;
}

// The normalisation factor of a term: its non-wildcard count, or 1 when it has none (ctcWordSpotMultiple).
template <typename Tok> FA_HD int non_wildcard_count(Tok tok, int n) {
    int k = 0;
    for (int i = 0; i < n; ++i) k += tok(i) != kWildcard;
    return k;
}

} // namespace ctc
} // namespace fa
