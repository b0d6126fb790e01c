// C ABI of CTC decoding (declared in include/fluidaudio_b200_ctc_decode.h): ctcGreedyDecode, ctcBeamSearch and
// ARPALanguageModel over ctc_decode_kernels.cu.  Every argument is checked here, before any copy or launch; every entry
// point that returns a status returns through guard() (c_abi.h), and the handle-less ones lease the pooled call
// context (call_context.h).
#include "../../../include/fluidaudio_b200_ctc_decode.h"
#include "../c_abi.h"
#include "ctc_decode.h"

#include <climits>
#include <cmath>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <utility>
#include <vector>

struct fa_ctc_lm {
    fa::ctc_decode::Lm lm;
};
struct fa_ctc_decoder {
    fa::ctc_decode::Decoder decoder;
};

using namespace fa;
using namespace fa::ctc_decode;

namespace {

// `count` + 1 offsets from 0, non-decreasing; every span below `max_span` and the last offset below 2^62
bool offsets_ok(const int64_t *off, long long count, long long max_span) {
    if (!off || off[0] != 0) return false;
    for (long long i = 0; i < count; ++i)
        if (off[i + 1] < off[i] || off[i + 1] - off[i] > max_span || off[i + 1] > (1LL << 62)) return false;
    return true;
}

// An open-addressing table of `keys` (none kEmpty) with their values, probed as ctc_decode_core.cuh probes it
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

int lm_tables(int32_t W, const char *words, const int64_t *off, const int32_t *has_uni, const float *lp,
              const float *bo, int64_t NB, const int32_t *ctx, const int32_t *word, const float *blp, LmTables &t) {
    std::set<std::string> seen;
    std::vector<std::pair<unsigned long long, int>> children;
    std::map<std::pair<int, unsigned char>, int> child_of;
    t.node_word.assign(1, kNoWord);
    t.uni_log_prob.resize((size_t)W);
    t.uni_backoff.resize((size_t)W);
    for (int w = 0; w < W; ++w) {
        const std::string s(words + off[w], (size_t)(off[w + 1] - off[w]));
        if (!seen.insert(s).second) return refuse("fa_ctc_lm_create: word %d repeats an earlier word", w);
        if (has_uni[w] && (!std::isfinite(lp[w]) || !std::isfinite(bo[w])))
            return refuse("fa_ctc_lm_create: word %d has a non-finite unigram log-prob or backoff", w);
        t.uni_log_prob[(size_t)w] = has_uni[w] ? lp[w] : kUnkLogProb;
        t.uni_backoff[(size_t)w] = has_uni[w] ? bo[w] : 0.0f;
        int node = kLmRoot;
        for (unsigned char c : s) {
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
    std::set<std::pair<int, int>> pairs;
    std::vector<std::pair<unsigned long long, float>> bigrams;
    for (long long i = 0; i < NB; ++i) {
        if (ctx[i] < 0 || ctx[i] >= W || word[i] < 0 || word[i] >= W)
            return refuse("fa_ctc_lm_create: bigram %lld names a word outside [0, %d)", i, W);
        if (!std::isfinite(blp[i])) return refuse("fa_ctc_lm_create: bigram %lld has a non-finite log-prob", i);
        if (!pairs.insert({ctx[i], word[i]}).second)
            return refuse("fa_ctc_lm_create: bigram %lld repeats an earlier bigram", i);
        bigrams.emplace_back(((unsigned long long)(unsigned)ctx[i] << 32) | (unsigned)word[i], blp[i]);
    }
    hash_table(children, t.child_key, t.child_node);
    hash_table(bigrams, t.bigram_key, t.bigram_log_prob);
    return FA_OK;
}

int beam_search(fa_ctc_decoder *h, const fa_ctc_lm *lm, bool on_device, const float *log_probs,
                const int64_t *row_offsets, int32_t clips, const fa_ctc_beam_config *cfg, int64_t *lengths,
                float *scores, int32_t *tokens, size_t cap, int64_t *total) {
    if (!h || !cfg || !total || clips < 0)
        return refuse("fa_ctc_beam_search: decoder, cfg or total is NULL or clip_count %d < 0", clips);
    if (!offsets_ok(row_offsets, clips, INT32_MAX))
        return refuse("fa_ctc_beam_search: row_offsets must be %lld offsets from 0, non-decreasing, each clip below "
                      "2^31 rows", (long long)clips + 1);
    const Decoder &d = h->decoder;
    const long long rows = row_offsets[clips];
    if (clips > 0 && (!lengths || !scores)) return refuse("fa_ctc_beam_search: lengths or scores is NULL");
    if (rows > 0 && !log_probs) return refuse("fa_ctc_beam_search: log_probs is NULL with %lld rows", rows);
    if (cap > 0 && !tokens) return refuse("fa_ctc_beam_search: tokens is NULL with capacity %lld", capacity(cap));
    if (cfg->beam_width < 0 || cfg->token_candidates < 0)
        return refuse("fa_ctc_beam_search: beam_width %d and token_candidates %d must be >= 0", cfg->beam_width,
                      cfg->token_candidates);
    if (lm && (!std::isfinite(cfg->lm_weight) || !std::isfinite(cfg->word_bonus)))
        return refuse("fa_ctc_beam_search: lm_weight and word_bonus must be finite");
    if (lm && lm->lm.device != d.device)
        return refuse("fa_ctc_beam_search: the LM is on device %d, the decoder on device %d", lm->lm.device, d.device);
    const int columns = d.vocab - (d.blank_id >= 0 && d.blank_id < d.vocab ? 1 : 0);
    const int k_eff = cfg->token_candidates < columns ? cfg->token_candidates : columns;
    if (cfg->beam_width > kMaxBeamWidth || k_eff > kMaxTokenCandidates) {
        set_error("fa_ctc_beam_search: beam_width %d and %d candidate tokens; at most %d and %d are supported",
                  cfg->beam_width, k_eff, kMaxBeamWidth, kMaxTokenCandidates);
        return FA_STATUS_UNSUPPORTED;
    }
    for (int b = 0; b < clips; ++b)
        if (2 * (row_offsets[b + 1] - row_offsets[b]) * cfg->beam_width + 1 >= INT32_MAX) {
            set_error("fa_ctc_beam_search: clip %d has more prefixes than a 31-bit node id holds", b);
            return FA_STATUS_INDEX_OVERFLOW;
        }
    return h->decoder.beam_search(lm ? &lm->lm : nullptr, on_device, log_probs, row_offsets, clips, cfg->beam_width,
                                  k_eff, cfg->lm_weight, cfg->word_bonus, lengths, scores, tokens, capacity(cap),
                                  total);
}

int greedy_call(bool on_device, const float *log_probs, const int64_t *row_offsets, int32_t clips, int32_t vocab,
                int32_t blank_id, int64_t *lengths, int32_t *tokens, size_t cap, int64_t *total) {
    if (!total || clips < 0 || vocab < 1)
        return refuse("fa_ctc_greedy: total is NULL, clip_count %d < 0 or vocab_size %d < 1", clips, vocab);
    if (!offsets_ok(row_offsets, clips, INT32_MAX))
        return refuse("fa_ctc_greedy: row_offsets must be %lld offsets from 0, non-decreasing, each clip below 2^31 "
                      "rows", (long long)clips + 1);
    const long long rows = row_offsets[clips];
    if (clips > 0 && !lengths) return refuse("fa_ctc_greedy: lengths is NULL");
    if (rows > 0 && !log_probs) return refuse("fa_ctc_greedy: log_probs is NULL with %lld rows", rows);
    if (cap > 0 && !tokens) return refuse("fa_ctc_greedy: tokens is NULL with capacity %lld", capacity(cap));
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) {
        return ctc_decode::greedy(C, on_device, log_probs, row_offsets, clips, vocab, blank_id, lengths, tokens,
                                  capacity(cap), total);
    });
}

} // namespace

FA_API void fa_ctc_beam_default_config(fa_ctc_beam_config *cfg) {
    if (cfg) *cfg = fa_ctc_beam_config{100, 40, 0.3f, 0.0f};
}

FA_API fa_status fa_ctc_lm_create(int32_t word_count, const char *words, const int64_t *word_offsets,
                                  const int32_t *has_unigram, const float *log_prob, const float *backoff,
                                  int64_t bigram_count, const int32_t *bigram_context, const int32_t *bigram_word,
                                  const float *bigram_log_prob, fa_ctc_lm **out) {
    return guard(__func__, [&]() -> int {
        if (!out) return refuse("fa_ctc_lm_create: out is NULL");
        *out = nullptr;
        if (word_count < 0 || bigram_count < 0)
            return refuse("fa_ctc_lm_create: word_count %d and bigram_count %lld must be >= 0", word_count,
                          (long long)bigram_count);
        if (!offsets_ok(word_offsets, word_count, INT32_MAX))
            return refuse("fa_ctc_lm_create: word_offsets must be %lld offsets from 0, non-decreasing",
                          (long long)word_count + 1);
        if ((word_offsets[word_count] > 0 && !words) ||
            (word_count > 0 && (!has_unigram || !log_prob || !backoff)) ||
            (bigram_count > 0 && (!bigram_context || !bigram_word || !bigram_log_prob)))
            return refuse("fa_ctc_lm_create: a required array is NULL (%d words, %lld bigrams)", word_count,
                          (long long)bigram_count);
        if (word_offsets[word_count] >= (1LL << 30) || bigram_count >= (1LL << 30)) {
            set_error("fa_ctc_lm_create: %lld word bytes and %lld bigrams, at most 2^30 - 1 each",
                      (long long)word_offsets[word_count], (long long)bigram_count);
            return FA_STATUS_INDEX_OVERFLOW;
        }
        LmTables t;
        const int st = lm_tables(word_count, words, word_offsets, has_unigram, log_prob, backoff, bigram_count,
                                 bigram_context, bigram_word, bigram_log_prob, t);
        if (st != FA_OK) return st;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        std::unique_ptr<fa_ctc_lm> h(new fa_ctc_lm());
        const int s2 = h->lm.init(t);
        if (s2 != FA_OK) return s2;
        *out = h.release();
        return FA_STATUS_OK;
    });
}

FA_API void fa_ctc_lm_destroy(fa_ctc_lm *lm) { delete lm; }

FA_API fa_status fa_ctc_decoder_create(int32_t vocab_size, int32_t blank_id, const char *pieces,
                                       const int64_t *piece_offsets, fa_ctc_decoder **out) {
    return guard(__func__, [&]() -> int {
        if (!out) return refuse("fa_ctc_decoder_create: out is NULL");
        *out = nullptr;
        if (vocab_size < 1) return refuse("fa_ctc_decoder_create: vocab_size %d must be >= 1", vocab_size);
        if (!offsets_ok(piece_offsets, vocab_size, INT32_MAX))
            return refuse("fa_ctc_decoder_create: piece_offsets must be %lld offsets from 0, non-decreasing",
                          (long long)vocab_size + 1);
        if (piece_offsets[vocab_size] > 0 && !pieces)
            return refuse("fa_ctc_decoder_create: pieces is NULL with %lld bytes", (long long)piece_offsets[vocab_size]);
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        std::unique_ptr<fa_ctc_decoder> h(new fa_ctc_decoder());
        const int st = h->decoder.init(vocab_size, blank_id, pieces, piece_offsets);
        if (st != FA_OK) return st;
        *out = h.release();
        return FA_STATUS_OK;
    });
}

FA_API void fa_ctc_decoder_destroy(fa_ctc_decoder *decoder) { delete decoder; }

FA_API fa_status fa_ctc_beam_search(fa_ctc_decoder *decoder, const fa_ctc_lm *lm, const float *log_probs,
                                    const int64_t *row_offsets, int32_t clip_count, const fa_ctc_beam_config *cfg,
                                    int64_t *lengths, float *scores, int32_t *tokens, size_t capacity,
                                    int64_t *total) {
    return guard(__func__, [&] {
        return beam_search(decoder, lm, false, log_probs, row_offsets, clip_count, cfg, lengths, scores, tokens,
                           capacity, total);
    });
}

FA_API fa_status fa_ctc_beam_search_device(fa_ctc_decoder *decoder, const fa_ctc_lm *lm, const float *d_log_probs,
                                           const int64_t *row_offsets, int32_t clip_count,
                                           const fa_ctc_beam_config *cfg, int64_t *lengths, float *scores,
                                           int32_t *d_tokens, size_t capacity, int64_t *total) {
    return guard(__func__, [&] {
        return beam_search(decoder, lm, true, d_log_probs, row_offsets, clip_count, cfg, lengths, scores, d_tokens,
                           capacity, total);
    });
}

FA_API fa_status fa_ctc_greedy(const float *log_probs, const int64_t *row_offsets, int32_t clip_count,
                               int32_t vocab_size, int32_t blank_id, int64_t *lengths, int32_t *tokens,
                               size_t capacity, int64_t *total) {
    return guard(__func__, [&] {
        return greedy_call(false, log_probs, row_offsets, clip_count, vocab_size, blank_id, lengths, tokens, capacity,
                           total);
    });
}

FA_API fa_status fa_ctc_greedy_device(const float *d_log_probs, const int64_t *row_offsets, int32_t clip_count,
                                      int32_t vocab_size, int32_t blank_id, int64_t *lengths, int32_t *d_tokens,
                                      size_t capacity, int64_t *total) {
    return guard(__func__, [&] {
        return greedy_call(true, d_log_probs, row_offsets, clip_count, vocab_size, blank_id, lengths, d_tokens,
                           capacity, total);
    });
}
