/* C ABI of CTC keyword spotting in libfluidaudio_b200.so, beside the main header it builds on (status codes).  Plain
 * C11, like the other headers under include/. */
#ifndef FLUIDAUDIO_B200_CTC_H
#define FLUIDAUDIO_B200_CTC_H

#include "fluidaudio_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* CTC keyword spotting (CTC-WS, custom-vocabulary boosting): CtcKeywordSpotter and CtcDPAlgorithm
 * (Sources/FluidAudio/ASR/Parakeet/SlidingWindow/CustomVocabulary/WordSpotting/) from the CTC model's logits to the
 * detections of every vocabulary term in every clip.  The CTC model and the tokenizers stay with the caller.  Frame
 * counts are int32: a clip or a matrix has fewer than 2^31 rows.  Every argument is checked before any copy or launch,
 * and a refused call changes nothing.  The _device variants take the float arrays in HBM and are asynchronous on the
 * call's stream unless stated otherwise; every other array is host memory.
 *
 * fa_ctc_log_softmax: applyLogSoftmax / makeLogProbs (CtcKeywordSpotter.swift:268-306, +Inference.swift:350-431).
 * logits is [frames x vocab] (FA_CTC_LAYOUT_TIME_MAJOR) or [vocab x frames] (FA_CTC_LAYOUT_VOCAB_MAJOR, the rank-4
 * CoreML output [1, V, 1, T]); log_probs is [frames x vocab], time-major.  Per row: x / temperature when the
 * temperature is not 1, the max, the float32 sum of exp(x - max) in index order, (x - max) - log(sum), and blank_bias
 * subtracted from column blank_id when the bias is non-zero and blank_id < vocab (a negative blank_id with a non-zero
 * bias is refused: the reference traps on it).  exp and log are (float)exp((double)x) and (float)log((double)x).
 * One launch, one thread per row.
 *
 * fa_ctc_merge_chunks: the concatenation of computeLogProbsChunked (+Inference.swift:96-126).  chunks holds the
 * chunk matrices [rows x vocab] back to back, chunk c at rows row_offsets[c] .. row_offsets[c+1] (chunk_count + 1
 * non-decreasing offsets from 0).  Empty chunks are skipped; the first non-empty chunk is taken whole, and each later
 * one averages min(overlap_frames, rows so far, its rows) of its first rows into the last rows so far
 * ((m + log(exp(a - m) + exp(b - m))) - 0.69314718, -inf where max(a, b) is) and appends the rest.  *frames receives
 * the joined row count; out [*frames x vocab] (out_len elements) too small gives FA_STATUS_OUTPUT_TOO_SMALL with
 * *frames set.  One launch.
 *
 * fa_ctc_spotter_create: the vocabulary in HBM.  Term k has the token ids tokens[term_offsets[k] ..
 * term_offsets[k+1]) (term_count + 1 non-decreasing offsets from 0); FA_CTC_WILDCARD matches any frame at no cost.
 * Ids outside [0, vocab_size) are accepted and keep the reference's meaning: such a token emits -FLT_MAX and such a
 * blank emits 0.  A term of more than FA_CTC_MAX_TERM_TOKENS tokens is refused with FA_STATUS_UNSUPPORTED (its 2N + 1
 * expanded states must fit one warp of 32 lanes x 8 states).  An empty term never matches.
 *
 * fa_ctc_spot: spotKeywordsFromLogProbs (CtcKeywordSpotter.swift:191-254) without its text-length filter, for
 * clip_count clips at once.  Clip b is log_probs rows row_offsets[b] .. row_offsets[b+1) ([rows x vocab_size]).
 * Term k of n tokens is held to min_score ? *min_score - max(0, n - 3) * 1.0 : -15 (no per-token relaxation without a
 * base, :218-222) and searched with ctcWordSpotMultiple (CtcDPAlgorithm.swift:311-392), overlapping detections merged.
 * counts[b * term_count + k] receives the detections of (clip b, term k) and *total their sum; detections receives
 * them in the reference's order: clip, then term, then merged order, each {clip, term, score, start_frame,
 * end_frame}.  capacity < *total gives FA_STATUS_OUTPUT_TOO_SMALL with counts and *total set and the detections
 * untouched.  One call is TWO kernel launches whatever the clip and term counts (the dynamic program with each pair's
 * merge, then the compaction; the compaction is skipped when *total is 0 or capacity too small) and one
 * synchronisation for the counts.  fa_ctc_spot_device takes log_probs and detections in HBM and returns after that
 * synchronisation with the compaction still queued on the spotter's stream; counts stays host memory.  A spotter is
 * not thread-safe.
 *
 * fa_ctc_spot_constrained: ctcWordSpotConstrained (CtcDPAlgorithm.swift:250-300) for query_count independent queries
 * over one [frames x vocab_size] matrix, in one launch.  Query q has the tokens tokens[token_offsets[q] ..
 * token_offsets[q+1]) (at most FA_CTC_MAX_TERM_TOKENS, FA_STATUS_UNSUPPORTED beyond) and the window search_start[q] ..
 * search_end[q], clamped to 0 .. frames as the reference clamps it.  Outputs per query: the score normalised by its
 * non-wildcard count (raw when there is none) and the global start and end frames; an empty window, one shorter than
 * the query or an empty query gives (-inf, clamped start, clamped start).  start_frame and end_frame are int64 because
 * the clamped start of a window past the end is returned as it is.  The host variant returns after one
 * synchronisation; the _device variant takes log_probs and the three outputs in HBM. */
#define FA_CTC_WILDCARD (-1)
#define FA_CTC_MAX_TERM_TOKENS 127

enum { FA_CTC_LAYOUT_TIME_MAJOR = 0, FA_CTC_LAYOUT_VOCAB_MAJOR = 1 };

typedef struct {
    int32_t clip, term;
    float score;
    int32_t start_frame, end_frame;
} fa_ctc_detection;
typedef struct fa_ctc_spotter fa_ctc_spotter;

fa_status fa_ctc_log_softmax(const float *logits, int32_t frames, int32_t vocab, int32_t layout, float temperature,
                             float blank_bias, int32_t blank_id, float *log_probs);
fa_status fa_ctc_log_softmax_device(const float *d_logits, int32_t frames, int32_t vocab, int32_t layout,
                                    float temperature, float blank_bias, int32_t blank_id, float *d_log_probs);
fa_status fa_ctc_merge_chunks(const float *chunks, const int64_t *row_offsets, int32_t chunk_count, int32_t vocab,
                              int32_t overlap_frames, float *out, size_t out_len, int32_t *frames);
fa_status fa_ctc_merge_chunks_device(const float *d_chunks, const int64_t *row_offsets, int32_t chunk_count,
                                     int32_t vocab, int32_t overlap_frames, float *d_out, size_t out_len,
                                     int32_t *frames);
fa_status fa_ctc_spotter_create(int32_t vocab_size, int32_t blank_id, int32_t term_count, const int32_t *tokens,
                                const int64_t *term_offsets, fa_ctc_spotter **out);
void fa_ctc_spotter_destroy(fa_ctc_spotter *h);
fa_status fa_ctc_spot(fa_ctc_spotter *h, const float *log_probs, const int64_t *row_offsets, int32_t clip_count,
                      const float *min_score, int64_t *counts, int64_t *total, fa_ctc_detection *detections,
                      size_t capacity);
fa_status fa_ctc_spot_device(fa_ctc_spotter *h, const float *d_log_probs, const int64_t *row_offsets,
                             int32_t clip_count, const float *min_score, int64_t *counts, int64_t *total,
                             fa_ctc_detection *d_detections, size_t capacity);
fa_status fa_ctc_spot_constrained(const float *log_probs, int32_t frames, int32_t vocab_size, int32_t blank_id,
                                  int32_t query_count, const int32_t *tokens, const int64_t *token_offsets,
                                  const int64_t *search_start, const int64_t *search_end, float *score,
                                  int64_t *start_frame, int64_t *end_frame);
fa_status fa_ctc_spot_constrained_device(const float *d_log_probs, int32_t frames, int32_t vocab_size,
                                         int32_t blank_id, int32_t query_count, const int32_t *tokens,
                                         const int64_t *token_offsets, const int64_t *search_start,
                                         const int64_t *search_end, float *d_score, int64_t *d_start_frame,
                                         int64_t *d_end_frame);

#ifdef __cplusplus
}
#endif
#endif /* FLUIDAUDIO_B200_CTC_H */
