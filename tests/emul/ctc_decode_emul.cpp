// Host run of CTC decoding's arithmetic (fluidaudio_b200/csrc/ctc_decode/ctc_decode_core.cuh; CPU test-suite only), in
// the kernels' own formulation: the frame's candidate tokens picked one at a time by ranks_before (topk_kernel), then
// per frame each beam's prelude, the order keys of its extension slots, its keep slot with the parent's extension
// folded in (generation index lowered, extension slot dead), the beam_width smallest keys in key order, the survivors'
// states with new prefixes consed into the clip's open-addressing trie and the LM trie walked (beam_kernel); the
// greedy argmax as the fold argmax_kernel reduces and the keep rule of collapse_kernel.  The LM tables are laid out and
// probed as fa_ctc_lm_create lays them out.
//   ctc_decode_emul_greedy(lp, T, V, blank, out) -> count
//   ctc_decode_emul_beam(lp, T, V, blank, pieces, piece_off, has_lm, <LM arrays>, B, K, weight, bonus, out, cap, score)
#include "../../fluidaudio_b200/csrc/ctc_decode/ctc_decode_core.cuh"

#include <algorithm>
#include <climits>
#include <cmath>
#include <map>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

using namespace fa::ctc_decode;

namespace {

template <typename V>
void hash_table(const std::vector<std::pair<unsigned long long, V>> &kv, std::vector<unsigned long long> &keys,
                std::vector<V> &vals) {
    const size_t cap = 2 * kv.size() + 1;
    keys.assign(cap, kEmpty);
    vals.assign(cap, V{});
    for (const auto &e : kv) {
        size_t s = (size_t)home_slot(e.first, (long long)cap);
        while (keys[s] != kEmpty) s = s + 1 == cap ? 0 : s + 1;
        keys[s] = e.first;
        vals[s] = e.second;
    }
}

struct LmHost {
    std::vector<unsigned long long> child_key, bigram_key;
    std::vector<int> child_node, node_word;
    std::vector<float> uni_lp, uni_bo, bigram_lp;
    LmView view() const {
        return LmView{child_key.data(), child_node.data(), (long long)child_key.size(), node_word.data(),
                      uni_lp.data(), uni_bo.data(), bigram_key.data(), bigram_lp.data(), (long long)bigram_key.size()};
    }
};

LmHost make_lm(int W, const char *words, const int64_t *off, const int32_t *has_uni, const float *lp, const float *bo,
               long long NB, const int32_t *ctx, const int32_t *word, const float *blp) {
    LmHost t;
    std::vector<std::pair<unsigned long long, int>> children;
    std::map<std::pair<int, unsigned char>, int> child_of;
    t.node_word.assign(1, kNoWord);
    for (int w = 0; w < W; ++w) {
        t.uni_lp.push_back(has_uni[w] ? lp[w] : kUnkLogProb);
        t.uni_bo.push_back(has_uni[w] ? bo[w] : 0.0f);
        int node = kLmRoot;
        for (long long i = off[w]; i < off[w + 1]; ++i) {
            const unsigned char c = (unsigned char)words[i];
            auto it = child_of.find({node, c});
            if (it == child_of.end()) {
                const int n = (int)t.node_word.size();
                t.node_word.push_back(kNoWord);
                it = child_of.emplace(std::make_pair(node, c), n).first;
                children.emplace_back(((unsigned long long)(unsigned)node << 8) | c, n);
            }
            node = it->second;
        }
        t.node_word[(size_t)node] = w;
    }
    std::vector<std::pair<unsigned long long, float>> bigrams;
    for (long long i = 0; i < NB; ++i)
        bigrams.emplace_back(((unsigned long long)(unsigned)ctx[i] << 32) | (unsigned)word[i], blp[i]);
    hash_table(children, t.child_key, t.child_node);
    hash_table(bigrams, t.bigram_key, t.bigram_lp);
    t.uni_lp.push_back(0.0f);
    t.uni_bo.push_back(0.0f);
    return t;
}

} // namespace

extern "C" {

int ctc_decode_emul_greedy(const float *lp, int T, int V, int blank, int *out) {
    int n = 0;
    for (int t = 0, prev = kNoToken; t < T; ++t) {
        const float *x = lp + (size_t)t * V;
        float bv = -INFINITY;
        int bi = INT_MAX;
        for (int v = 0; v < V; ++v)
            if (!std::isnan(x[v]) && (bi == INT_MAX || greedy_better(x[v], v, bv, bi))) {
                bv = x[v];
                bi = v;
            }
        const int id = bi == INT_MAX || std::isnan(x[0]) ? 0 : bi;
        if (greedy_keep(id, prev, blank)) out[n++] = id;
        prev = id;
    }
    return n;
}

long long ctc_decode_emul_beam(const float *lp, int T, int V, int blank, const char *pieces, const int64_t *piece_off,
                               int has_lm, int W, const char *words, const int64_t *word_off, const int32_t *has_uni,
                               const float *ulp, const float *ubo, long long NB, const int32_t *bctx,
                               const int32_t *bword, const float *blp, int B, int K_req, float weight, float bonus,
                               int *out, long long cap_out, float *score) {
    const int columns = V - (blank >= 0 && blank < V ? 1 : 0);
    const int K = std::min(K_req, columns), KK = K + 1;
    LmHost lm_host;
    LmView view{};
    if (has_lm) {
        lm_host = make_lm(W, words, word_off, has_uni, ulp, ubo, NB, bctx, bword, blp);
        view = lm_host.view();
    }
    const LmView *lm = has_lm ? &view : nullptr;
    std::vector<long long> off64(piece_off, piece_off + V + 1);
    std::vector<unsigned char> boundary((size_t)V);
    for (int v = 0; v < V; ++v) {
        const unsigned char *p = reinterpret_cast<const unsigned char *>(pieces) + piece_off[v];
        boundary[(size_t)v] = piece_off[v + 1] - piece_off[v] >= 3 && p[0] == 0xE2 && p[1] == 0x96 && p[2] == 0x81;
    }
    const Pieces pc{reinterpret_cast<const unsigned char *>(pieces), off64.data(), boundary.data()};
    const long long cap = 2LL * T * B + 1;
    std::vector<unsigned long long> trie((size_t)cap, kEmpty);
    auto cas = [&](long long s, unsigned long long e, unsigned long long d) {
        const unsigned long long old = trie[(size_t)s];
        if (old == e) trie[(size_t)s] = d;
        return old;
    };
    std::vector<Beam> cur{Beam{0.0f, -INFINITY, 0.0f, kRootNode, -1, kNoToken, 0, kLmRoot, kNoWord}};
    std::vector<int> top_id((size_t)K);
    std::vector<float> top_lp((size_t)K);
    for (int t = 0; t < T && !cur.empty(); ++t) {
        const float *x = lp + (size_t)t * V;
        const float blank_lp = blank >= 0 && blank < V ? x[blank] : -INFINITY;
        for (int r = 0; r < K; ++r) {   // topk_kernel's rounds: the best column after the previous pick
            int bi = -1;
            float bv = 0.0f;
            for (int v = 0; v < V; ++v) {
                if (v == blank || (r > 0 && !ranks_before(top_lp[(size_t)r - 1], top_id[(size_t)r - 1], x[v], v)))
                    continue;
                if (bi < 0 || ranks_before(x[v], v, bv, bi)) {
                    bv = x[v];
                    bi = v;
                }
            }
            top_id[(size_t)r] = bi;
            top_lp[(size_t)r] = bv;
        }
        const int nb = (int)cur.size(), n = nb * KK;
        std::vector<Prelude> pre((size_t)nb);
        std::unordered_map<int, int> beam_of;
        for (int i = 0; i < nb; ++i) {
            pre[(size_t)i] = prelude(cur[(size_t)i], lm, weight, bonus);
            beam_of[cur[(size_t)i].node] = i;
        }
        std::vector<unsigned long long> keys((size_t)n, kEmpty);
        for (int s = 0; s < n; ++s) {
            const int i = s / KK, c = s - i * KK;
            if (c == 0) continue;
            const int v = top_id[(size_t)c - 1];
            const float pnb = ext_pnb(cur[(size_t)i], pre[(size_t)i], v, top_lp[(size_t)c - 1]);
            keys[(size_t)s] = order_key(beam_total(-INFINITY, pnb, ext_lm(cur[(size_t)i], pre[(size_t)i], boundary[(size_t)v] != 0)), s, s);
        }
        std::vector<float> keep_pb((size_t)nb), keep_pnb((size_t)nb);
        int merged = 0;
        for (int i = 0; i < nb; ++i) {
            const Beam &b = cur[(size_t)i];
            int rc = -1;
            for (int c = 0; c < K && b.last >= 0; ++c)
                if (top_id[(size_t)c] == b.last) rc = c;
            float pb, pnb;
            keep_start(b, pre[(size_t)i], blank_lp, rc >= 0, rc >= 0 ? top_lp[(size_t)rc] : 0.0f, pb, pnb);
            int gen = i * KK;
            if (rc >= 0 && b.parent >= 0) {
                auto it = beam_of.find(b.parent);
                if (it != beam_of.end()) {
                    const int j = it->second;
                    pnb = log_add_exp(pnb, ext_pnb(cur[(size_t)j], pre[(size_t)j], b.last, top_lp[(size_t)rc]));
                    const int slot = j * KK + 1 + rc;
                    gen = std::min(gen, slot);
                    keys[(size_t)slot] = kEmpty;
                    ++merged;
                }
            }
            keep_pb[(size_t)i] = pb;
            keep_pnb[(size_t)i] = pnb;
            keys[(size_t)i * KK] = order_key(beam_total(pb, pnb, b.lm), gen, i * KK);
        }
        std::vector<unsigned long long> live;
        for (unsigned long long k : keys)
            if (k != kEmpty) live.push_back(k);
        if ((int)live.size() != n - merged) return -1;   // a merge the kernels would count differently
        std::sort(live.begin(), live.end());
        live.resize((size_t)std::min<long long>(B, (long long)live.size()));
        std::vector<Beam> next;
        for (unsigned long long k : live) {
            const int slot = key_slot(k), i = slot / KK, c = slot - i * KK;
            const Beam &b = cur[(size_t)i];
            Beam nb_;
            if (c == 0) {
                nb_ = b;
                nb_.pb = keep_pb[(size_t)i];
                nb_.pnb = keep_pnb[(size_t)i];
            } else {
                const int v = top_id[(size_t)c - 1];
                nb_ = ext_beam(b, pre[(size_t)i], v, ext_pnb(b, pre[(size_t)i], v, top_lp[(size_t)c - 1]), lm, pc);
                nb_.node = cons(trie.data(), cap, b.node, v, cas);
            }
            next.push_back(nb_);
        }
        cur = std::move(next);
    }
    if (cur.empty()) {
        *score = -INFINITY;
        return 0;
    }
    int best = 0;
    std::vector<float> tot(cur.size());
    for (size_t i = 0; i < cur.size(); ++i) tot[i] = final_total(cur[i], lm, weight, bonus);
    for (size_t i = 1; i < cur.size(); ++i)
        if (tot[i] > tot[(size_t)best]) best = (int)i;
    const Beam &b = cur[(size_t)best];
    *score = tot[(size_t)best];
    int node = b.node;
    for (int k = b.len - 1; k >= 0; --k) {
        if (k < cap_out) out[k] = node_token(trie.data(), node);
        node = node_parent(trie.data(), node);
    }
    return b.len;
}

} // extern "C"
