// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
//
// Sequential CPU restatement of CTC keyword spotting: CtcKeywordSpotter.applyLogSoftmax / makeLogProbs
// (CtcKeywordSpotter.swift:268-306, +Inference.swift:350-431), mergeOverlapFrame and the chunk concatenation
// (+Inference.swift:96-126, :329-346) and CtcDPAlgorithm (CtcDPAlgorithm.swift:121-392): fillDPTable with its full
// (T+1) x (2N+1) tables, ctcWordSpotConstrained and ctcWordSpotMultiple, written from the reference's description and
// not from the kernels' rolling formulation.  Built with -O2 -ffp-contract=off (oracle_ctc.py), so every float
// operation is one IEEE operation; exp and log are the correctly rounded float32 functions of oracle_float.h, the
// library's definition in place of Apple's closed libm.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <vector>

#include "oracle_float.h"

namespace {

const float kNegMax = -FLT_MAX;
const int kWildcard = -1;

float fexp(float x) { return oracle_float::exp32(x); }
float flog(float x) { return oracle_float::log32(x); }

enum Kind { kBlank, kToken, kWild };
struct Sym {
    Kind kind;
    int id;
};

std::vector<Sym> expanded(const int *tok, int n) {
    std::vector<Sym> s;
    for (int i = 0; i < n; ++i) {
        s.push_back({kBlank, 0});
        s.push_back(tok[i] == kWildcard ? Sym{kWild, 0} : Sym{kToken, tok[i]});
    }
    s.push_back({kBlank, 0});
    return s;
}

float emission(const Sym &s, const float *frame, int V, int blank) {
    switch (s.kind) {
    case kBlank: return blank >= 0 && blank < V ? frame[blank] : 0.0f;
    case kToken: return s.id >= 0 && s.id < V ? frame[s.id] : kNegMax;
    default: return 0.0f;
    }
}

bool can_skip(const std::vector<Sym> &s, int i) {
    if (i < 2) return false;
    if (s[i].kind == kBlank) return false;
    if (s[i].kind == kToken) return !(s[i - 2].kind == kToken && s[i - 2].id == s[i].id);
    return s[i - 2].kind != kWild;
}

struct Tables {
    std::vector<std::vector<float>> dp;   // [T+1][N+1]
    std::vector<std::vector<int>> back, last;
};

Tables fill(const float *lp, int T, int V, const int *tok, int N, int blank) {
    Tables r;
    r.dp.assign(T + 1, std::vector<float>(N + 1, kNegMax));
    r.back.assign(T + 1, std::vector<int>(N + 1, 0));
    r.last.assign(T + 1, std::vector<int>(N + 1, 0));
    for (int t = 0; t <= T; ++t) r.dp[t][0] = 0.0f;
    if (N == 0) return r;
    const std::vector<Sym> s = expanded(tok, N);
    const int L = (int)s.size();
    std::vector<std::vector<float>> d(T + 1, std::vector<float>(L, kNegMax));
    std::vector<std::vector<int>> st(T + 1, std::vector<int>(L, 0)), lt(T + 1, std::vector<int>(L, 0));
    for (int t = 0; t <= T; ++t) {
        d[t][0] = 0.0f;
        st[t][0] = t;
    }
    for (int t = 1; t <= T; ++t) {
        const float *frame = lp + (size_t)(t - 1) * V;
        for (int i = 1; i < L; ++i) {
            const float e = emission(s[i], frame, V, blank);
            const bool wild = s[i].kind == kWild, tokn = s[i].kind == kToken;
            const float added = wild ? 0.0f : e;
            const float stay = d[t - 1][i], adv = d[t - 1][i - 1];
            const float skip = can_skip(s, i) ? d[t - 1][i - 2] : kNegMax;
            float best = stay;
            int kind = 0;
            if (adv > best) {
                best = adv;
                kind = 1;
            }
            if (skip > best) {
                best = skip;
                kind = 2;
            }
            if (best <= kNegMax / 2) {
                d[t][i] = kNegMax;
                continue;
            }
            d[t][i] = best + added;
            const bool match = tokn || wild;
            if (kind == 0) {
                st[t][i] = st[t - 1][i];
                lt[t][i] = match ? t : lt[t - 1][i];
            } else if (kind == 1) {
                st[t][i] = i == 1 ? t - 1 : st[t - 1][i - 1];
                lt[t][i] = match ? t : lt[t - 1][i - 1];
            } else {
                st[t][i] = st[t - 1][i - 2];
                lt[t][i] = match ? t : lt[t - 1][i - 2];
            }
        }
    }
    for (int t = 0; t <= T; ++t)
        for (int n = 1; n <= N; ++n) {
            const int a = 2 * n - 1, b = 2 * n;
            const float sa = a < L ? d[t][a] : kNegMax, sb = b < L ? d[t][b] : kNegMax;
            if (sa >= sb) {
                r.dp[t][n] = sa;
                r.back[t][n] = st[t][a];
                r.last[t][n] = lt[t][a];
            } else {
                r.dp[t][n] = sb;
                r.back[t][n] = st[t][b];
                r.last[t][n] = lt[t][b];
            }
        }
    return r;
}

int non_wildcard(const int *tok, int n) {
    int k = 0;
    for (int i = 0; i < n; ++i) k += tok[i] != kWildcard;
    return k;
}

struct Cand {
    float score;
    int start, end;
};

} // namespace

extern "C" {

void oracle_ctc_log_softmax(const float *x, int T, int V, int layout, float temperature, float bias, int blank,
                            float *out) {
    std::vector<float> row(V);
    for (int t = 0; t < T; ++t) {
        for (int v = 0; v < V; ++v) row[v] = layout == 1 ? x[(size_t)v * T + t] : x[(size_t)t * V + v];
        if (temperature != 1.0f)
            for (float &e : row) e = e / temperature;
        float m = row[0];
        for (int v = 1; v < V; ++v)
            if (m < row[v]) m = row[v];
        float sum = 0.0f;
        for (int v = 0; v < V; ++v) sum += fexp(row[v] - m);
        const float lse = flog(sum);
        float *o = out + (size_t)t * V;
        for (int v = 0; v < V; ++v) o[v] = (row[v] - m) - lse;
        if (bias != 0.0f && blank < V) o[blank] -= bias;
    }
}

// out holds at least the input rows; returns the joined row count
long long oracle_ctc_merge_chunks(const float *chunks, const int64_t *offsets, int count, int V, int overlap,
                                  float *out) {
    long long rows = 0;
    for (int c = 0; c < count; ++c) {
        const long long n = offsets[c + 1] - offsets[c];
        if (n == 0) continue;
        const float *src = chunks + (size_t)offsets[c] * V;
        long long ov = 0;
        if (rows > 0) {
            ov = std::min<long long>(std::min<long long>(overlap, rows), n);
            for (long long i = 0; i < ov; ++i) {
                float *e = out + (size_t)(rows - ov + i) * V;
                const float *in = src + (size_t)i * V;
                for (int j = 0; j < V; ++j) {
                    const float a = e[j], b = in[j];
                    const float m = b >= a ? b : a;
                    e[j] = m == -INFINITY ? -INFINITY : m + flog(fexp(a - m) + fexp(b - m)) - 0.69314718f;
                }
            }
        }
        for (long long i = ov; i < n; ++i, ++rows)
            for (int j = 0; j < V; ++j) out[(size_t)rows * V + j] = src[(size_t)i * V + j];
    }
    return rows;
}

void oracle_ctc_constrained(const float *lp, int T, int V, const int *tok, int N, int64_t search_start,
                            int64_t search_end, int blank, float *score, int64_t *start, int64_t *end) {
    const long long cs = std::max<long long>(0, search_start), ce = std::min<long long>(T, search_end);
    if (N == 0 || ce <= cs || ce - cs < N) {
        *score = -INFINITY;
        *start = *end = cs;
        return;
    }
    const int W = (int)(ce - cs);
    const Tables r = fill(lp + (size_t)cs * V, W, V, tok, N, blank);
    int best_end = 0;
    float best = kNegMax;
    for (int t = N; t <= W; ++t)
        if (r.dp[t][N] > best) {
            best = r.dp[t][N];
            best_end = t;
        }
    const int norm = non_wildcard(tok, N);
    *score = norm > 0 ? best / (float)norm : best;
    *start = cs + r.back[best_end][N];
    *end = cs + r.last[best_end][N];
}

// ctcWordSpotMultiple with mergeOverlap; writes at most `cap` detections, returns their count
int oracle_ctc_multiple(const float *lp, int T, int V, const int *tok, int N, float min_score, int blank, float *score,
                        int *start, int *end, int cap) {
    if (N == 0 || T == 0) return 0;
    const Tables r = fill(lp, T, V, tok, N, blank);
    const int nw = non_wildcard(tok, N);
    const float norm = nw > 0 ? (float)nw : 1.0f;
    if (T < N) return 0;
    std::vector<Cand> c;
    for (int t = N; t <= T; ++t) {
        const float s = r.dp[t][N] / norm;
        const float prev = t > N ? r.dp[t - 1][N] / norm : kNegMax;
        const float next = t < T ? r.dp[t + 1][N] / norm : kNegMax;
        if (s >= prev && s > next && s >= min_score) c.push_back({s, r.back[t][N], r.last[t][N]});
    }
    if (c.empty()) {
        int be = 0;
        float bs = kNegMax;
        for (int t = N; t <= T; ++t) {
            const float s = r.dp[t][N] / norm;
            if (s > bs) {
                bs = s;
                be = t;
            }
        }
        if (bs >= min_score) c.push_back({bs, r.back[be][N], r.last[be][N]});
    }
    std::stable_sort(c.begin(), c.end(), [](const Cand &a, const Cand &b) { return a.start < b.start; });
    std::vector<Cand> m;
    for (const Cand &x : c) {
        if (!m.empty() && x.start <= m.back().end) {
            Cand best = x.score > m.back().score ? x : m.back();
            best.end = std::max(m.back().end, x.end);
            m.back() = best;
        } else {
            m.push_back(x);
        }
    }
    const int n = (int)std::min<size_t>(m.size(), (size_t)cap);
    for (int i = 0; i < n; ++i) {
        score[i] = m[i].score;
        start[i] = m[i].start;
        end[i] = m[i].end;
    }
    return (int)m.size();
}

float oracle_ctc_threshold(int has_base, float base, int n) {
    if (!has_base) return -15.0f;
    return base - (float)std::max(0, n - 3) * 1.0f;
}

int oracle_ctc_non_wildcard_count(const int *tok, int n) { return non_wildcard(tok, n); }

} // extern "C"
