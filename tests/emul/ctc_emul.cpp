// Host run of CTC keyword spotting's arithmetic (fluidaudio_b200/csrc/ctc/ctc_core.cuh; CPU test-suite only), in the
// kernels' own formulation: one row at a time for the log-softmax, one column fold for the chunk merge, and for the
// dynamic program one rolling row of expanded states updated from the highest state down (as a warp's lanes update
// their registers), the candidate scan one frame behind and the in-place sort and merge of lane 0.
//   ctc_emul_log_softmax(x, T, V, layout, temperature, bias, blank, out)
//   ctc_emul_merge_overlap(a, b, n, out)                     out[i] = mergeOverlapFrame column i
//   ctc_emul_multiple(lp, T, V, tok, N, threshold, blank, score, start, end, cap) -> merged count
//   ctc_emul_constrained(lp, T, V, tok, N, search_start, search_end, blank, score, start, end)
//   ctc_emul_threshold(has_base, base, n)
#include "../../fluidaudio_b200/csrc/ctc/ctc_core.cuh"

#include <algorithm>
#include <cstdint>
#include <vector>

using namespace fa::ctc;

namespace {

// the kernels' warp_dp, lane by lane in one row; on_frame(t, dp[t][N])
template <typename F> void rolling_dp(const float *lp, int T, int V, const int *tok, int N, int blank, F on_frame) {
    const int L = 2 * N + 1;
    auto tk = [&](int i) { return tok[i]; };
    std::vector<State> st(L);
    std::vector<Cell> c(L, Cell{kNeg, 0, 0});
    for (int s = 0; s < L; ++s) st[s] = expanded_state(s, tk, V, blank);
    c[0] = Cell{0.0f, 0, 0};
    for (int t = 1; t <= T; ++t) {
        const float *row = lp + (size_t)(t - 1) * V;
        for (int s = L - 1; s >= 1; --s)
            c[s] = step_cell(c[s], c[s - 1], s >= 2 ? c[s - 2] : c[0], st[s], emission(st[s], row), t, s);
        c[0] = Cell{0.0f, t, 0};
        on_frame(t, project(c[2 * N - 1], c[2 * N]));
    }
}

} // namespace

extern "C" {

void ctc_emul_log_softmax(const float *x, int T, int V, int layout, float temperature, float bias, int blank,
                          float *out) {
    for (long long t = 0; t < T; ++t) {
        const long long step = layout == 1 ? T : 1;
        const float *src = x + (layout == 1 ? t : t * V);
        float *dst = out + t * V;
        log_softmax_row(V, temperature, bias, blank, [&](int v) { return src[v * step]; },
                        [&](int v, float r) { dst[v] = r; });
    }
}

void ctc_emul_merge_overlap(const float *a, const float *b, long long n, float *out) {
    for (long long i = 0; i < n; ++i) out[i] = merge_overlap(a[i], b[i]);
}

int ctc_emul_multiple(const float *lp, int T, int V, const int *tok, int N, float threshold, int blank, float *score,
                      int *start, int *end, int cap) {
    if (N == 0 || T < N) return 0;
    std::vector<Candidate> c((size_t)(T / 2 + 2));
    const int nw = non_wildcard_count([&](int i) { return tok[i]; }, N);
    Scan scan;
    scan.init(nw > 0 ? (float)nw : 1.0f, threshold);
    int n = 0;
    auto emit = [&](const Candidate &x) { c[(size_t)n++] = x; };
    rolling_dp(lp, T, V, tok, N, blank, [&](int t, const Cell &cell) {
        if (t >= N) scan.push(cell, emit);
    });
    scan.finish(emit);
    n = merge_candidates(c.data(), n);
    for (int i = 0; i < std::min(n, cap); ++i) {
        score[i] = c[(size_t)i].score;
        start[i] = c[(size_t)i].start;
        end[i] = c[(size_t)i].end;
    }
    return n;
}

void ctc_emul_constrained(const float *lp, int T, int V, const int *tok, int N, int64_t search_start,
                          int64_t search_end, int blank, float *score, int64_t *start, int64_t *end) {
    const long long cs = std::max<long long>(0, search_start), ce = std::min<long long>(T, search_end);
    const long long W = ce > cs ? ce - cs : 0;
    if (N == 0 || W < N) {
        *score = -INFINITY;
        *start = *end = cs;
        return;
    }
    Cell best{kNeg, 0, 0};
    rolling_dp(lp + (size_t)cs * V, (int)W, V, tok, N, blank, [&](int t, const Cell &cell) {
        if (t >= N && cell.dp > best.dp) best = cell;
    });
    const int norm = non_wildcard_count([&](int i) { return tok[i]; }, N);
    *score = norm > 0 ? fa::fp::f_div(best.dp, (float)norm) : best.dp;
    *start = cs + best.start;
    *end = cs + best.last;
}

float ctc_emul_threshold(int has_base, float base, int n) { return term_threshold(has_base != 0, base, n); }

} // extern "C"
