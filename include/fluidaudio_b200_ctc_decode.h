/* C ABI of CTC decoding in libfluidaudio_b200.so, beside the main header it builds on (status codes).  Plain C11, like
 * the other headers under include/. */
#ifndef FLUIDAUDIO_B200_CTC_DECODE_H
#define FLUIDAUDIO_B200_CTC_DECODE_H

#include "fluidaudio_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* CTC decoding: ctcGreedyDecode, ctcBeamSearch and ARPALanguageModel
 * (Sources/FluidAudio/ASR/Parakeet/SlidingWindow/CTC/) from the CTC model's log-probs to token ids, for many clips per
 * call.  decodeCtcTokenIds (ids to text) stays with the caller.  Clip b is log_probs rows row_offsets[b] ..
 * row_offsets[b+1) of a [rows x vocab] time-major matrix (clip_count + 1 non-decreasing offsets from 0, each clip below
 * 2^31 rows).  Outputs are the ids of each clip back to back in clip order: lengths[b] ids of clip b, *total in all.
 * capacity (in ids) below *total gives FA_STATUS_OUTPUT_TOO_SMALL with lengths, *total (and scores) set and tokens
 * untouched.  Every argument is checked before any copy or launch, and a refused call changes nothing.  The _device
 * variants take log_probs and tokens in HBM and return after the one synchronisation with the last copy still queued
 * on the call's stream; every other array is host memory.  Floats are float32; exp and log are
 * (float)exp((double)x) and (float)log((double)x).
 *
 * fa_ctc_greedy: ctcGreedyDecode([[Float]]) (CtcDecoder.swift:15-36).  Per row the first maximum (a later column
 * replaces the best only when strictly greater, so a NaN wins only in column 0); the row's id is kept when it is not
 * blank_id and differs from the previous row's id (the blank counts as a previous id).  A blank_id outside
 * [0, vocab_size) never matches.  At most three launches (argmax per row, the per-clip collapse, the gather; the gather
 * is skipped when *total is 0 or the capacity short) and one synchronisation, on a pooled call context.
 *
 * fa_ctc_lm_create: an ARPALanguageModel in HBM on the current device, its values already natural-log (the log10 of
 * the file times Float(log(10.0))).  Word w is the UTF-8 bytes words[word_offsets[w] .. word_offsets[w+1])
 * (word_count + 1 non-decreasing offsets from 0): every unigram, bigram context and bigram target, each once.
 * has_unigram[w] != 0 gives it the unigram (log_prob[w], backoff[w]); bigram i is P(bigram_word[i] |
 * bigram_context[i]) = bigram_log_prob[i].  Refused: duplicate words or bigrams, indices outside [0, word_count), and
 * non-finite values.  score(word, prev) is the bigram [prev][word] when it exists, else backoff(prev) + logProb(word)
 * with backoff 0 when prev is nil or has no unigram and logProb -23.026 (unkLogProb) when word has none.  An LM is
 * read-only: decoders on its device may share it.
 *
 * fa_ctc_decoder_create: the piece table of a vocabulary in HBM on the current device, with the stream and scratch its
 * searches use (the scratch grows as needed).  Token v (0 .. vocab_size - 1) is the UTF-8 piece pieces[
 * piece_offsets[v] .. piece_offsets[v+1]); an id the vocabulary lacks has the empty piece.  A piece that starts with
 * U+2581 starts a word.  A decoder is not thread-safe.
 *
 * fa_ctc_beam_search: ctcBeamSearch([[Float]]) (CtcDecoder.swift:118-241), prefix beam search with the Graves repeat
 * rule and, with an lm, word-level LM terms lm_weight * score + word_bonus at each completed word and for the trailing
 * one.  Ties, which the reference breaks by hash order, are broken by first insertion: the candidates of a frame are
 * the blank extension of each beam, then per candidate token its repeat-same and its extension; the prune keeps the
 * beam_width best totals, the earlier inserted first among equals, in that order; the result is the first best total.
 * A frame's candidate tokens are its token_candidates best columns (blank_id left out, ties to the lower index);
 * token_candidates beyond the non-blank columns takes them all.  scores[b] receives the best total of clip b: 0 for a
 * clip of no rows, -inf with no ids when beam_width is 0.  A NaN or +inf log-prob gives FA_STATUS_INVALID_ARGUMENT and
 * leaves every output untouched (checked on the device, read at the synchronisation).  beam_width above
 * FA_CTC_DECODE_MAX_BEAM_WIDTH, or more than FA_CTC_DECODE_MAX_TOKEN_CANDIDATES candidate tokens, is
 * FA_STATUS_UNSUPPORTED: a frame's at most 128 x 65 candidates then fit one CTA's shared memory.  A non-finite
 * lm_weight or word_bonus is refused.  Three launches (the top-K per row, the beam search per clip, the gather; the
 * top-K is skipped without rows, the gather when *total is 0 or the capacity short) and one synchronisation, on the
 * decoder's stream; the lm must be on the decoder's device.  One clip is one CTA walking its frames in order. */
#define FA_CTC_DECODE_MAX_BEAM_WIDTH 128
#define FA_CTC_DECODE_MAX_TOKEN_CANDIDATES 64

typedef struct {
    int32_t beam_width;         /* beamWidth, default 100 */
    int32_t token_candidates;   /* tokenCandidates, default 40 */
    float lm_weight;            /* lmWeight (alpha), default 0.3 */
    float word_bonus;           /* wordBonus (beta, nats), default 0 */
} fa_ctc_beam_config;

typedef struct fa_ctc_lm fa_ctc_lm;
typedef struct fa_ctc_decoder fa_ctc_decoder;

void fa_ctc_beam_default_config(fa_ctc_beam_config *cfg);
fa_status fa_ctc_lm_create(int32_t word_count, const char *words, const int64_t *word_offsets,
                           const int32_t *has_unigram, const float *log_prob, const float *backoff,
                           int64_t bigram_count, const int32_t *bigram_context, const int32_t *bigram_word,
                           const float *bigram_log_prob, fa_ctc_lm **out);
void fa_ctc_lm_destroy(fa_ctc_lm *lm);
fa_status fa_ctc_decoder_create(int32_t vocab_size, int32_t blank_id, const char *pieces,
                                const int64_t *piece_offsets, fa_ctc_decoder **out);
void fa_ctc_decoder_destroy(fa_ctc_decoder *decoder);
fa_status fa_ctc_beam_search(fa_ctc_decoder *decoder, const fa_ctc_lm *lm, const float *log_probs,
                             const int64_t *row_offsets, int32_t clip_count, const fa_ctc_beam_config *cfg,
                             int64_t *lengths, float *scores, int32_t *tokens, size_t capacity, int64_t *total);
fa_status fa_ctc_beam_search_device(fa_ctc_decoder *decoder, const fa_ctc_lm *lm, const float *d_log_probs,
                                    const int64_t *row_offsets, int32_t clip_count, const fa_ctc_beam_config *cfg,
                                    int64_t *lengths, float *scores, int32_t *d_tokens, size_t capacity,
                                    int64_t *total);
fa_status fa_ctc_greedy(const float *log_probs, const int64_t *row_offsets, int32_t clip_count, int32_t vocab_size,
                        int32_t blank_id, int64_t *lengths, int32_t *tokens, size_t capacity, int64_t *total);
fa_status fa_ctc_greedy_device(const float *d_log_probs, const int64_t *row_offsets, int32_t clip_count,
                               int32_t vocab_size, int32_t blank_id, int64_t *lengths, int32_t *d_tokens,
                               size_t capacity, int64_t *total);

#ifdef __cplusplus
}
#endif
#endif /* FLUIDAUDIO_B200_CTC_DECODE_H */
