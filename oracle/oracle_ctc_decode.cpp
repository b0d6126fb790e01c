// ORACLE — TEST INFRASTRUCTURE ONLY.  Sequential CPU restatement of CTC decoding (CtcDecoder.swift,
// ARPALanguageModel.swift): ctcGreedyDecode, ctcBeamSearch with its LM terms, ARPALanguageModel.score and logAddExp.
// Prefixes are ids of a consed trie ((parent, token) -> id), beams an insertion-ordered map (a vector with an index by
// prefix id), the prune a stable sort: the reference's code with insertion-ordered dictionaries.  Words are byte
// strings.  exp and log are (float)exp((double)x) and (float)log((double)x); built with -ffp-contract=off.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

namespace {

const float kUnk = -23.026f;
const std::string kBoundary = "\xE2\x96\x81";

float f_exp(float x) { return (float)std::exp((double)x); }
float f_log(float x) { return (float)std::log((double)x); }

float log_add_exp(float a, float b) {
    if (a == -INFINITY) return b;
    if (b == -INFINITY) return a;
    const float m = b >= a ? b : a;   // Swift.max
    return m + f_log(f_exp(a - m) + f_exp(b - m));
}

struct Lm {
    std::map<std::string, std::pair<float, float>> unigrams;
    std::map<std::string, std::map<std::string, float>> bigrams;

    float score(const std::string &word, bool has_prev, const std::string &prev) const {
        if (has_prev) {
            auto c = bigrams.find(prev);
            if (c != bigrams.end()) {
                auto w = c->second.find(word);
                if (w != c->second.end()) return w->second;
            }
        }
        float backoff = 0.0f;
        if (has_prev) {
            auto u = unigrams.find(prev);
            if (u != unigrams.end()) backoff = u->second.second;
        }
        auto u = unigrams.find(word);
        return backoff + (u != unigrams.end() ? u->second.first : kUnk);
    }
};

Lm make_lm(int W, const char *words, const int64_t *off, const int32_t *has_uni, const float *lp, const float *bo,
           long long NB, const int32_t *ctx, const int32_t *word, const float *blp) {
    Lm lm;
    std::vector<std::string> w((size_t)W);
    for (int i = 0; i < W; ++i) {
        w[(size_t)i].assign(words + off[i], (size_t)(off[i + 1] - off[i]));
        if (has_uni[i]) lm.unigrams[w[(size_t)i]] = {lp[i], bo[i]};
    }
    for (long long i = 0; i < NB; ++i) lm.bigrams[w[(size_t)ctx[i]]][w[(size_t)word[i]]] = blp[i];
    return lm;
}

struct Beam {
    int node, last;
    float pb, pnb, lm;
    std::string partial;   // wordPieces.joined()
    bool has_prev;
    std::string prev;
    float total() const { return log_add_exp(pb, pnb) + lm; }
};

} // namespace

extern "C" {

float oracle_ctc_log_add_exp(float a, float b) { return log_add_exp(a, b); }

int oracle_ctc_greedy(const float *lp, int T, int V, int blank, int *out) {
    int n = 0, prev = -1;
    for (int t = 0; t < T && V > 0; ++t) {
        const float *f = lp + (size_t)t * V;
        int best = 0;
        float bv = f[0];
        for (int v = 1; v < V; ++v)
            if (f[v] > bv) {
                bv = f[v];
                best = v;
            }
        if (best != blank && best != prev) out[n++] = best;
        prev = best;
    }
    return n;
}

float oracle_ctc_lm_score(int W, const char *words, const int64_t *off, const int32_t *has_uni, const float *lp,
                          const float *bo, long long NB, const int32_t *ctx, const int32_t *word, const float *blp,
                          const char *w, long long wn, int has_prev, const char *p, long long pn) {
    const Lm lm = make_lm(W, words, off, has_uni, lp, bo, NB, ctx, word, blp);
    return lm.score(std::string(w, (size_t)wn), has_prev != 0, has_prev ? std::string(p, (size_t)pn) : std::string());
}

// ctcBeamSearch over one clip [T x V]: the best prefix's ids into out (at most cap), its total into *score; returns its
// length.  *recreated counts extensions that re-made a prefix which was pruned while a child of it is still a beam.
long long oracle_ctc_beam(const float *lp, int T, int V, int blank, const char *pieces, const int64_t *piece_off,
                          int has_lm, int W, const char *words, const int64_t *word_off, const int32_t *has_uni,
                          const float *ulp, const float *ubo, long long NB, const int32_t *bctx, const int32_t *bword,
                          const float *blp, int B, int K, float weight, float bonus, int *out, long long cap,
                          float *score, long long *recreated) {
    Lm lm;
    if (has_lm) lm = make_lm(W, words, word_off, has_uni, ulp, ubo, NB, bctx, bword, blp);
    std::vector<std::string> piece((size_t)V);
    for (int v = 0; v < V; ++v) piece[(size_t)v].assign(pieces + piece_off[v], (size_t)(piece_off[v + 1] - piece_off[v]));
    std::map<std::pair<int, int>, int> trie;   // (parent, token) -> node
    std::vector<int> parent{-1}, token{-1};
    std::vector<Beam> beams{Beam{0, -1, 0.0f, -INFINITY, 0.0f, "", false, ""}};
    *recreated = 0;
    std::vector<int> cols;
    for (int t = 0; t < T; ++t) {
        const float *f = lp + (size_t)t * V;
        const float blank_lp = blank >= 0 && blank < V ? f[blank] : -INFINITY;
        cols.clear();
        for (int v = 0; v < V; ++v)
            if (v != blank) cols.push_back(v);
        std::stable_sort(cols.begin(), cols.end(), [&](int a, int b) { return f[a] > f[b]; });
        if ((int)cols.size() > K) cols.resize((size_t)K);
        std::vector<Beam> next;
        std::unordered_map<int, size_t> at;
        std::unordered_map<int, bool> beam_node, beam_parent;
        for (const Beam &b : beams) {
            beam_node[b.node] = true;
            beam_parent[parent[(size_t)b.node]] = true;
        }
        auto merge = [&](const Beam &b) {
            auto it = at.find(b.node);
            if (it == at.end()) {
                at[b.node] = next.size();
                next.push_back(b);
            } else {
                Beam &e = next[it->second];
                e.pb = log_add_exp(e.pb, b.pb);
                e.pnb = log_add_exp(e.pnb, b.pnb);
            }
        };
        for (const Beam &beam : beams) {
            const float prev_total = log_add_exp(beam.pb, beam.pnb);
            Beam blank_beam = beam;
            blank_beam.pb = prev_total + blank_lp;
            blank_beam.pnb = -INFINITY;
            merge(blank_beam);
            for (int v : cols) {
                const float tok = f[v];
                const std::string &pc = piece[(size_t)v];
                std::string partial = beam.partial, prev = beam.prev;
                bool has_prev = beam.has_prev;
                float delta = 0.0f;
                if (has_lm && pc.compare(0, kBoundary.size(), kBoundary) == 0) {
                    const bool done = !partial.empty();
                    delta = done ? weight * lm.score(partial, has_prev, prev) + bonus : 0.0f;
                    if (done) {
                        prev = partial;
                        has_prev = true;
                    }
                    partial = pc.substr(kBoundary.size());
                } else if (has_lm) {
                    partial += pc;
                }
                const auto key = std::make_pair(beam.node, v);
                auto it = trie.find(key);
                int node;
                if (it == trie.end()) {
                    node = (int)parent.size();
                    trie[key] = node;
                    parent.push_back(beam.node);
                    token.push_back(v);
                } else {
                    node = it->second;
                    if (!beam_node.count(node) && beam_parent.count(node)) ++*recreated;
                }
                if (beam.last == v) {
                    Beam same = beam;
                    same.pb = -INFINITY;
                    same.pnb = beam.pnb + tok;
                    merge(same);
                    merge(Beam{node, v, -INFINITY, beam.pb + tok, beam.lm + delta, partial, has_prev, prev});
                } else {
                    merge(Beam{node, v, -INFINITY, prev_total + tok, beam.lm + delta, partial, has_prev, prev});
                }
            }
        }
        std::stable_sort(next.begin(), next.end(), [](const Beam &a, const Beam &b) { return a.total() > b.total(); });
        if ((int)next.size() > B) next.resize((size_t)B);
        beams = std::move(next);
    }
    if (beams.empty()) {
        *score = -INFINITY;
        return 0;
    }
    size_t best = 0;
    float best_total = 0.0f;
    for (size_t i = 0; i < beams.size(); ++i) {
        Beam b = beams[i];
        if (has_lm && !b.partial.empty()) b.lm += weight * lm.score(b.partial, b.has_prev, b.prev) + bonus;
        const float tot = b.total();
        if (i == 0 || best_total < tot) {
            best = i;
            best_total = tot;
        }
    }
    std::vector<int> ids;
    for (int n = beams[best].node; n != 0; n = parent[(size_t)n]) ids.push_back(token[(size_t)n]);
    std::reverse(ids.begin(), ids.end());
    for (size_t i = 0; i < ids.size() && (long long)i < cap; ++i) out[i] = ids[i];
    *score = best_total;
    return (long long)ids.size();
}

} // extern "C"
