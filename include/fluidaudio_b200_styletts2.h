/* StyleTTS2 synthesis around the caller's models (Sources/FluidAudio/TTS/StyleTTS2/Pipeline/Synthesize/
 * StyleTTS2Synthesizer.swift:33-133, glue in StyleTTS2GlueOps.swift, constants in StyleTTS2Constants.swift): the host
 * work synthesize does between its eight model stages, for many requests per launch.  The text encoder, bert, ref
 * encoder, fused sampler, duration predictor, f0n/har source, decoder_pre and decoder_upsample stay with the caller.
 *
 * A request's life, one call each (no request outlives a call, so there is no handle):
 *   fa_styletts2_plan            the bert / sampler bucket for its token count
 *   fa_styletts2_sampler_inputs  bert's padded tokens and attention mask, the fused sampler's seeded noise
 *   fa_styletts2_style           the alpha / beta blend of s_pred and ref_s into ref and s
 *   fa_styletts2_align           durations from the duration predictor's logits, then en and asr for f0n/har and
 *                                decoder_pre
 * Slicing bert's d_en to realN columns, the all-zero text masks and the 50-sample tail trim are views the caller takes.
 *
 * Every data-taking call has a host variant, which returns after its synchronisation, and a _device variant, whose bulk
 * arrays are HBM and which is asynchronous on the library's pooled call stream except where noted.  Offsets, per-request
 * scalars, token counts, frames, durations and reasons stay host arrays.  Every call checks every request and argument
 * before any copy or launch; a refused call writes nothing but the reasons (and, for FA_STATUS_OUTPUT_TOO_SMALL, the
 * frames).  Launch counts are given for count > 0.
 *
 * Arithmetic (DESIGN §4.15):
 *   noise      StyleTTS2NoiseSource, the same implementation as fa_luxtts_begin's noise (include/fluidaudio_b200_luxtts.h):
 *              equal to a sequential float64 evaluation bit for bit, except where the float64 value lies within 2^-40
 *              (relative) of a float32 rounding midpoint, where the neighbouring float32 is allowed.
 *   blend      ref = a p + (1 - a) r, s = b p' + (1 - b) r': 1 - a in float32, each product and sum rounded
 *              separately (Swift does not contract).  Bit for bit.
 *   durations  sum += 1 / (1 + expf(-x)) in float32 over channels 0 .. C-1, each operation rounded separately, with
 *              expf evaluated as float64 exp rounded once to float32 (the correctly rounded value up to midpoint
 *              cases; Apple's expf is closed and unpinned), then roundf (half away from zero) and max(., 1).  A NaN
 *              logit makes the sum NaN: Swift's Int(NaN) traps, so the call is refused with
 *              FA_STYLETTS2_NONFINITE_DURATION.  Durations equal a float64-exp oracle's except where an exp value lies
 *              within 2^-40 of a float32 midpoint and that flips a rounding.
 *   expansion  en[c, f] = 0.0f + d[tok(max(f - 1, 0)), c] and asr[c, f] = 0.0f + t_en[c, tok(max(f - 1, 0))], where
 *              tok(g) is the token whose prefix interval of durations holds frame g: the one-hot alignment matmul, the
 *              transpose and the HiFi-GAN shift in one pass.  This is netlib sgemm with beta = 0 (C is zeroed, zero
 *              entries of B are skipped): -0 becomes +0, inf and NaN pass through, and a non-finite value of another
 *              token does not reach the frame.  Every finite non-zero value is what any sgemm gives; the sign of a
 *              zero and non-finite values elsewhere in a row are unpinned against Accelerate's cblas_sgemm.  NaN
 *              payloads are not kept.
 */
#ifndef FLUIDAUDIO_B200_STYLETTS2_H
#define FLUIDAUDIO_B200_STYLETTS2_H

#include "fluidaudio_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define FA_STYLETTS2_STYLE_DIM 256       /* StyleTTS2Constants.styleDim */
#define FA_STYLETTS2_REF_SPLIT 128       /* StyleTTS2Constants.refSplit */
#define FA_STYLETTS2_NOISE_ROWS 5        /* StyleTTS2Constants.diffusionSteps: noise_init and 4 noises_aux rows */
#define FA_STYLETTS2_DEFAULT_TOKENS 57   /* StyleTTS2Constants.defaultBertTokens */
#define FA_STYLETTS2_MAX_TOKENS 256      /* the largest of StyleTTS2Constants.bucketTokenSizes {64, 128, 256} */
#define FA_STYLETTS2_TAIL_TRIM 50        /* StyleTTS2Constants.tailTrimSamples */
#define FA_STYLETTS2_SAMPLE_RATE 24000   /* StyleTTS2Constants.sampleRate */

/* Reason codes of a refused request. */
enum {
    FA_STYLETTS2_OK = 0,
    FA_STYLETTS2_NO_TOKENS = 1,           /* no token: the reference divides by realN = 0 */
    FA_STYLETTS2_NO_BUCKET = 2,           /* more than 256 tokens: StyleTTS2Error.noBucketAvailable */
    FA_STYLETTS2_NONFINITE_DURATION = 3   /* a NaN duration logit: Int(NaN) traps in roundDurations */
};

/* The bert / fused-sampler bucket of a request of token_count tokens: 57 for 1 .. 57, then 64, 128, 256.  0 tokens is
 * FA_STYLETTS2_NO_TOKENS and more than 256 FA_STYLETTS2_NO_BUCKET, with *bucket = 0.  A negative count is
 * FA_STATUS_INVALID_ARGUMENT.  No launch. */
fa_status fa_styletts2_plan(int32_t token_count, int32_t *bucket, int32_t *reason);

/* For `count` requests of one bucket: request i's token ids are token_ids[offsets[i] .. offsets[i+1]) (offsets
 * non-decreasing from offsets[0] >= 0) and its noise seed is seeds[i].  reasons[i] is set for every request; a request
 * of no bucket, or of a bucket other than `bucket`, refuses the call with FA_STATUS_INVALID_ARGUMENT.  Writes
 *   tokens          [count x bucket] int32  the ids, then 0
 *   attention_mask  [count x bucket] int32  1 for the ids, then 0
 *   noise           [count x 5 x 256]       Gaussians 0 .. 1279 of StyleTTS2NoiseSource(seeds[i]): row 0 is
 *                                           noise_init, rows 1 .. 4 are noises_aux
 * 1 launch. */
fa_status fa_styletts2_sampler_inputs(int32_t count, const int32_t *token_ids, const int64_t *offsets,
                                      const uint64_t *seeds, int32_t bucket, int32_t *tokens, int32_t *attention_mask,
                                      float *noise, int32_t *reasons);
fa_status fa_styletts2_sampler_inputs_device(int32_t count, const int32_t *d_token_ids, const int64_t *offsets,
                                             const uint64_t *seeds, int32_t bucket, int32_t *d_tokens,
                                             int32_t *d_attention_mask, float *d_noise, int32_t *reasons);

/* blendStyle for `count` requests: s_pred and ref_s [count x 256], alphas and betas [count] (host), ref and s
 * [count x 128].  ref = alpha s_pred[:128] + (1 - alpha) ref_s[:128], s = beta s_pred[128:] + (1 - beta) ref_s[128:].
 * 1 launch. */
fa_status fa_styletts2_style(int32_t count, const float *s_pred, const float *ref_s, const float *alphas,
                             const float *betas, float *ref, float *s);
fa_status fa_styletts2_style_device(int32_t count, const float *d_s_pred, const float *d_ref_s, const float *alphas,
                                    const float *betas, float *d_ref, float *d_s);

/* The duration-aligned decoder inputs of `count` requests; request i has n = token_counts[i] tokens (1 .. 256).
 *   logits  the duration predictor's [1, n, C]: token t's C >= 1 logits at
 *           logits + i * logit_request_stride + t * logit_row_stride (logit_row_stride >= C,
 *           logit_request_stride >= n * logit_row_stride)
 *   d       the duration predictor's [1, n, dC]: token t's channel c at d + i * d_request_stride + t * d_row_stride + c
 *           (d_row_stride >= dC, d_request_stride >= n * d_row_stride)
 *   t_en    the text encoder's [1, tC, n]: channel c's token t at t_en + i * t_en_request_stride + c * t_en_row_stride
 *           + t (t_en_row_stride >= n, t_en_request_stride >= tC * t_en_row_stride)
 * Launch 1 rounds the durations and sums them into F = frames[i]; the call synchronises and reads frames, durations
 * and the NaN flags.  A NaN logit sets reasons[i] = FA_STYLETTS2_NONFINITE_DURATION and refuses the call with
 * FA_STATUS_INVALID_ARGUMENT.  If any F > frame_stride, the call returns FA_STATUS_OUTPUT_TOO_SMALL with frames set.
 * Otherwise reasons[i] = 0, frames[i] = F, durations (NULL, or sum(token_counts) int32, request i's after the earlier
 * requests') are set and launch 2 writes
 *   en   [count x dC x frame_stride]  the expansion of d, zero from frame F on
 *   asr  [count x tC x frame_stride]  the expansion of t_en, zero from frame F on
 * dC and tC are 1 .. 2^20, C is 1 .. 2^24, frame_stride is 1 .. 2^22.  2 launches, 1 when refused after the
 * durations.  The _device variant synchronises once, between its launches. */
fa_status fa_styletts2_align(int32_t count, const int32_t *token_counts, const float *logits, int32_t logit_channels,
                             int64_t logit_row_stride, int64_t logit_request_stride, const float *d, int32_t d_channels,
                             int64_t d_row_stride, int64_t d_request_stride, const float *t_en, int32_t t_en_channels,
                             int64_t t_en_row_stride, int64_t t_en_request_stride, int64_t frame_stride, float *en,
                             float *asr, int64_t *frames, int32_t *durations, int32_t *reasons);
fa_status fa_styletts2_align_device(int32_t count, const int32_t *token_counts, const float *d_logits,
                                    int32_t logit_channels, int64_t logit_row_stride, int64_t logit_request_stride,
                                    const float *d_d, int32_t d_channels, int64_t d_row_stride,
                                    int64_t d_request_stride, const float *d_t_en, int32_t t_en_channels,
                                    int64_t t_en_row_stride, int64_t t_en_request_stride, int64_t frame_stride,
                                    float *d_en, float *d_asr, int64_t *frames, int32_t *durations, int32_t *reasons);

#ifdef __cplusplus
}
#endif

#endif /* FLUIDAUDIO_B200_STYLETTS2_H */
