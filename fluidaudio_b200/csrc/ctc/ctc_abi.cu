// C ABI of CTC keyword spotting (declared in include/fluidaudio_b200_ctc.h): CtcKeywordSpotter and CtcDPAlgorithm over
// ctc_kernels.cu.  Every argument is checked here, before any copy or launch; every entry point that returns a status
// returns through guard() (c_abi.h), and the handle-less ones lease the pooled call context (call_context.h).
#include "../../../include/fluidaudio_b200_ctc.h"
#include "c_abi.h"
#include "ctc_core.cuh"
#include "ctc_spot.h"

#include <algorithm>
#include <climits>
#include <memory>
#include <vector>

struct fa_ctc_spotter {
    fa::ctc::Spotter spotter;
};

using namespace fa;

namespace {

// `count` + 1 offsets from 0, non-decreasing; every span below `max_span` and the last offset below 2^62
bool offsets_ok(const int64_t *off, int count, long long max_span) {
    if (!off || off[0] != 0) return false;
    for (int i = 0; i < count; ++i)
        if (off[i + 1] < off[i] || off[i + 1] - off[i] > max_span || off[i + 1] > (1LL << 62)) return false;
    return true;
}

// The first term or query longer than the kernels support, or -1
int too_long(const int64_t *off, int count) {
    for (int i = 0; i < count; ++i)
        if (off[i + 1] - off[i] > ctc::kMaxTokens) return i;
    return -1;
}

int log_softmax(bool on_device, const float *logits, int32_t frames, int32_t vocab, int32_t layout,
                float temperature, float blank_bias, int32_t blank_id, float *log_probs) {
    if (frames < 0 || vocab < 0) return refuse("fa_ctc_log_softmax: frames %d and vocab %d must be >= 0", frames, vocab);
    if (layout != FA_CTC_LAYOUT_TIME_MAJOR && layout != FA_CTC_LAYOUT_VOCAB_MAJOR)
        return refuse("fa_ctc_log_softmax: layout %d is not a FA_CTC_LAYOUT_* value", layout);
    if (blank_bias != 0.0f && blank_id < 0)
        return refuse("fa_ctc_log_softmax: blank_id %d is negative with a non-zero blank bias", blank_id);
    if (frames == 0 || vocab == 0) return FA_STATUS_OK;
    if (!logits || !log_probs) return refuse("fa_ctc_log_softmax: logits or log_probs is NULL");
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) {
        return ctc::log_softmax(C, on_device, logits, frames, vocab, layout, temperature, blank_bias, blank_id,
                                log_probs);
    });
}

int merge_chunks(bool on_device, const float *chunks, const int64_t *row_offsets, int32_t chunk_count, int32_t vocab,
                 int32_t overlap_frames, float *out, size_t out_len, int32_t *frames) {
    if (chunk_count < 0 || vocab < 0 || overlap_frames < 0 || !frames)
        return refuse("fa_ctc_merge_chunks: chunk_count %d, vocab %d and overlap_frames must be >= 0 and frames "
                      "non-NULL", chunk_count, vocab);
    if (chunk_count > 0 && !offsets_ok(row_offsets, chunk_count, INT32_MAX))
        return refuse("fa_ctc_merge_chunks: row_offsets must be %lld offsets from 0, non-decreasing",
                      (long long)chunk_count + 1);
    const long long in_rows = chunk_count > 0 ? row_offsets[chunk_count] : 0;
    if (in_rows > INT32_MAX) return refuse("fa_ctc_merge_chunks: %lld rows, at most 2^31 - 1", in_rows);
    // each input row's output row (computeLogProbsChunked, +Inference.swift:99-126)
    std::vector<long long> dest((size_t)in_rows);
    long long rows = 0;
    for (int c = 0; c < chunk_count; ++c) {
        const long long n = row_offsets[c + 1] - row_offsets[c];
        if (n == 0) continue;
        const long long ov = std::min<long long>({(long long)overlap_frames, rows, n});
        for (long long i = 0; i < n; ++i) dest[(size_t)(row_offsets[c] + i)] = i < ov ? rows - ov + i : rows++;
    }
    if (rows * vocab > 0 && (!chunks || !out))
        return refuse("fa_ctc_merge_chunks: chunks or out is NULL");
    if (capacity(out_len) < rows * vocab) {
        *frames = (int32_t)rows;
        set_error("fa_ctc_merge_chunks: %lld output elements, out_len %lld", rows * vocab, capacity(out_len));
        return FA_STATUS_OUTPUT_TOO_SMALL;
    }
    *frames = (int32_t)rows;
    if (rows * vocab == 0) return FA_STATUS_OK;
    std::vector<long long> row_src((size_t)rows + 1, 0), src((size_t)in_rows);
    for (long long i = 0; i < in_rows; ++i) ++row_src[(size_t)dest[(size_t)i] + 1];
    for (long long r = 0; r < rows; ++r) row_src[(size_t)r + 1] += row_src[(size_t)r];
    std::vector<long long> fill(row_src.begin(), row_src.end() - 1);
    for (long long i = 0; i < in_rows; ++i) src[(size_t)fill[(size_t)dest[(size_t)i]]++] = i;
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) {
        return ctc::merge_chunks(C, on_device, chunks, in_rows, vocab, row_src, src, out);
    });
}

int spot(fa_ctc_spotter *h, bool on_device, const float *log_probs, const int64_t *row_offsets, int32_t clip_count,
         const float *min_score, int64_t *counts, int64_t *total, fa_ctc_detection *detections, size_t cap) {
    if (!h || !total || clip_count < 0) return refuse("fa_ctc_spot: h or total is NULL or clip_count %d < 0", clip_count);
    if (!offsets_ok(row_offsets, clip_count, INT32_MAX))
        return refuse("fa_ctc_spot: row_offsets must be %lld offsets from 0, non-decreasing, each clip below 2^31 "
                      "rows", (long long)clip_count + 1);
    const int K = h->spotter.terms;
    const long long pairs = (long long)clip_count * K, rows = row_offsets[clip_count];
    if (pairs > 0 && !counts) return refuse("fa_ctc_spot: counts is NULL with %lld pairs", pairs);
    if (rows > 0 && !log_probs) return refuse("fa_ctc_spot: log_probs is NULL with %lld rows", rows);
    if (cap > 0 && !detections) return refuse("fa_ctc_spot: detections is NULL with capacity %lld", capacity(cap));
    if ((long long)((K + 3) / 4) * clip_count > INT32_MAX) {
        set_error("fa_ctc_spot: %lld clips x %d terms is more than one launch holds", (long long)clip_count, K);
        return FA_STATUS_INDEX_OVERFLOW;
    }
    return h->spotter.spot(on_device, log_probs, row_offsets, clip_count, min_score, counts, total, detections,
                           capacity(cap));
}

int spot_constrained(bool on_device, const float *log_probs, int32_t frames, int32_t vocab, int32_t blank_id,
                     int32_t query_count, const int32_t *tokens, const int64_t *token_offsets,
                     const int64_t *search_start, const int64_t *search_end, float *score, int64_t *start_frame,
                     int64_t *end_frame) {
    if (frames < 0 || vocab < 1 || query_count < 0)
        return refuse("fa_ctc_spot_constrained: frames %d must be >= 0, vocab_size %d >= 1 and query_count >= 0",
                      frames, vocab);
    if (!offsets_ok(token_offsets, query_count, INT32_MAX) || token_offsets[query_count] > INT32_MAX)
        return refuse("fa_ctc_spot_constrained: token_offsets must be %lld offsets from 0, non-decreasing, below "
                      "2^31", (long long)query_count + 1);
    if (query_count == 0) return FA_STATUS_OK;
    if ((token_offsets[query_count] > 0 && !tokens) || !search_start || !search_end || !score || !start_frame ||
        !end_frame || ((long long)frames * vocab > 0 && !log_probs))
        return refuse("fa_ctc_spot_constrained: a required array is NULL (%lld queries)", query_count);
    const int q_long = too_long(token_offsets, query_count);
    if (q_long >= 0) {
        set_error("fa_ctc_spot_constrained: query %d has %lld tokens, at most %d are supported", q_long,
                  (long long)(token_offsets[q_long + 1] - token_offsets[q_long]), ctc::kMaxTokens);
        return FA_STATUS_UNSUPPORTED;
    }
    std::vector<ctc::QueryDesc> q((size_t)query_count);
    for (int i = 0; i < query_count; ++i) {
        const long long cs = std::max<long long>(0, search_start[i]), ce = std::min<long long>(frames, search_end[i]);
        q[(size_t)i] = ctc::QueryDesc{cs, ce > cs ? ce - cs : 0, (int)token_offsets[i],
                                      (int)(token_offsets[i + 1] - token_offsets[i])};
    }
    std::vector<int> tok(tokens, tokens + token_offsets[query_count]);
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) {
        return ctc::spot_constrained(C, on_device, log_probs, frames, vocab, blank_id, q, tok, score, start_frame,
                                     end_frame);
    });
}

} // namespace

FA_API fa_status fa_ctc_log_softmax(const float *logits, int32_t frames, int32_t vocab, int32_t layout,
                                    float temperature, float blank_bias, int32_t blank_id, float *log_probs) {
    return guard(__func__, [&] {
        return log_softmax(false, logits, frames, vocab, layout, temperature, blank_bias, blank_id, log_probs);
    });
}

FA_API fa_status fa_ctc_log_softmax_device(const float *d_logits, int32_t frames, int32_t vocab, int32_t layout,
                                           float temperature, float blank_bias, int32_t blank_id,
                                           float *d_log_probs) {
    return guard(__func__, [&] {
        return log_softmax(true, d_logits, frames, vocab, layout, temperature, blank_bias, blank_id, d_log_probs);
    });
}

FA_API fa_status fa_ctc_merge_chunks(const float *chunks, const int64_t *row_offsets, int32_t chunk_count,
                                     int32_t vocab, int32_t overlap_frames, float *out, size_t out_len,
                                     int32_t *frames) {
    return guard(__func__, [&] {
        return merge_chunks(false, chunks, row_offsets, chunk_count, vocab, overlap_frames, out, out_len, frames);
    });
}

FA_API fa_status fa_ctc_merge_chunks_device(const float *d_chunks, const int64_t *row_offsets, int32_t chunk_count,
                                            int32_t vocab, int32_t overlap_frames, float *d_out, size_t out_len,
                                            int32_t *frames) {
    return guard(__func__, [&] {
        return merge_chunks(true, d_chunks, row_offsets, chunk_count, vocab, overlap_frames, d_out, out_len, frames);
    });
}

FA_API fa_status fa_ctc_spotter_create(int32_t vocab_size, int32_t blank_id, int32_t term_count,
                                       const int32_t *tokens, const int64_t *term_offsets, fa_ctc_spotter **out) {
    return guard(__func__, [&]() -> int {
        if (!out) return refuse("fa_ctc_spotter_create: out is NULL");
        *out = nullptr;
        if (vocab_size < 1 || term_count < 0)
            return refuse("fa_ctc_spotter_create: vocab_size %d must be >= 1 and term_count %d >= 0", vocab_size,
                          term_count);
        if (!offsets_ok(term_offsets, term_count, INT32_MAX) || term_offsets[term_count] > INT32_MAX)
            return refuse("fa_ctc_spotter_create: term_offsets must be %lld offsets from 0, non-decreasing, below "
                          "2^31", (long long)term_count + 1);
        if (term_offsets[term_count] > 0 && !tokens)
            return refuse("fa_ctc_spotter_create: tokens is NULL with %lld tokens", term_offsets[term_count]);
        const int k_long = too_long(term_offsets, term_count);
        if (k_long >= 0) {
            set_error("fa_ctc_spotter_create: term %d has %lld tokens, at most %d are supported", k_long,
                      (long long)(term_offsets[k_long + 1] - term_offsets[k_long]), ctc::kMaxTokens);
            return FA_STATUS_UNSUPPORTED;
        }
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        std::unique_ptr<fa_ctc_spotter> h(new fa_ctc_spotter());
        const int st = h->spotter.init(vocab_size, blank_id, term_count, tokens, term_offsets);
        if (st != FA_OK) return st;
        *out = h.release();
        return FA_STATUS_OK;
    });
}

FA_API void fa_ctc_spotter_destroy(fa_ctc_spotter *h) { delete h; }

FA_API fa_status fa_ctc_spot(fa_ctc_spotter *h, const float *log_probs, const int64_t *row_offsets,
                             int32_t clip_count, const float *min_score, int64_t *counts, int64_t *total,
                             fa_ctc_detection *detections, size_t capacity) {
    return guard(__func__, [&] {
        return spot(h, false, log_probs, row_offsets, clip_count, min_score, counts, total, detections, capacity);
    });
}

FA_API fa_status fa_ctc_spot_device(fa_ctc_spotter *h, const float *d_log_probs, const int64_t *row_offsets,
                                    int32_t clip_count, const float *min_score, int64_t *counts, int64_t *total,
                                    fa_ctc_detection *d_detections, size_t capacity) {
    return guard(__func__, [&] {
        return spot(h, true, d_log_probs, row_offsets, clip_count, min_score, counts, total, d_detections, capacity);
    });
}

FA_API fa_status fa_ctc_spot_constrained(const float *log_probs, int32_t frames, int32_t vocab_size,
                                         int32_t blank_id, int32_t query_count, const int32_t *tokens,
                                         const int64_t *token_offsets, const int64_t *search_start,
                                         const int64_t *search_end, float *score, int64_t *start_frame,
                                         int64_t *end_frame) {
    return guard(__func__, [&] {
        return spot_constrained(false, log_probs, frames, vocab_size, blank_id, query_count, tokens, token_offsets,
                                search_start, search_end, score, start_frame, end_frame);
    });
}

FA_API fa_status fa_ctc_spot_constrained_device(const float *d_log_probs, int32_t frames, int32_t vocab_size,
                                                int32_t blank_id, int32_t query_count, const int32_t *tokens,
                                                const int64_t *token_offsets, const int64_t *search_start,
                                                const int64_t *search_end, float *d_score, int64_t *d_start_frame,
                                                int64_t *d_end_frame) {
    return guard(__func__, [&] {
        return spot_constrained(true, d_log_probs, frames, vocab_size, blank_id, query_count, tokens, token_offsets,
                                search_start, search_end, d_score, d_start_frame, d_end_frame);
    });
}
