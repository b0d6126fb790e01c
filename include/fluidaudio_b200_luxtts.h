/* LuxTTS synthesis around the caller's models (Sources/FluidAudio/TTS/LuxTts/LuxTtsSynthesizer.swift:46-299, arithmetic
 * in LuxTtsSolver.swift, constants in LuxTtsConstants.swift): everything synthesize does on the host between the text
 * encoder, the FmDecoder and the vocoder, for many requests per launch.  The models stay with the caller.
 *
 * A handle holds live requests.  Each request owns one slot in HBM: the float32 flow-matching state x in the
 * FmDecoder's [1024 x 100] layout, zero past features_length x 100.  A request's life:
 *   fa_luxtts_begin              plan, RMS, gain, prompt mel, speech_condition, padding_mask, noise x0 into the slot
 *   fa_luxtts_text_condition     token_embeds -> text_condition (any time after begin)
 *   4 x (fa_luxtts_model_inputs, the caller's FmDecoder, fa_luxtts_advance)
 *   fa_luxtts_vocoder_input      the vocoder's [100 x bucket] mel (step 4)
 *   fa_luxtts_finish             truncate, clip, rescale the vocoder's audio and close the request
 *
 * Every data-taking call has a host variant, which returns after one synchronisation, and a _device variant, whose
 * bulk arrays are HBM and which is asynchronous on the handle's stream (fa_luxtts_begin_device synchronises once, for
 * the silent-prompt check).  Request ids, offsets and per-request scalars stay host arrays.  Every call checks every
 * named request (open, none twice, the step it needs) and every argument before any copy or launch; a refused call
 * changes nothing.  Launch counts are given per call, for count > 0.
 *
 * Arithmetic (DESIGN §4.14):
 *   noise     StyleTTS2NoiseSource (SplitMix64; seed 0 means 0xdeadbeefcafebabe).  The state after draw k is
 *             s0 + k * 0x9e3779b97f4a7c15 (mod 2^64), so Gaussian j reads draws 2j+1 (u1) and 2j+2 (u2) directly.
 *             u = (z >> 11) / 2^53, u <= 0 becomes DBL_MIN, Float(sqrt(-2 log u1) * cos((2 pi) u2)) in float64, every
 *             operation rounded separately.  The device's float64 log and cos are not correctly rounded, so the float32
 *             result equals the host's bit for bit except where the float64 value lies within 2^-40 (relative) of a
 *             float32 rounding midpoint, where the neighbouring float32 is allowed.
 *   RMS       the mean square of the capped prompt, accumulated in float64 in one fixed tree (each of 256 lanes sums
 *             samples lane, lane + 256, ... in order, then a pairwise tree over the lanes), divided by n in float64,
 *             rounded once to float32, then sqrtf.  vDSP_measqv's order is unpinned.  gain = 0.1f / rms and its
 *             product with the prompt are float32; a prompt is boosted when rms < 0.1f.
 *   update    the float32 vDSP path of synthesize: x1p = v (1 - t) + x, x0p = v (-t) + x,
 *             x = x0p (1 - tNext) + x1p tNext, on the last step x = x1p; every product and sum rounded separately
 *             (unpinned against vDSP, whose fusing is not documented).  t = Float(timeSteps[step]), 1 - t in float32.
 *   clip      vDSP_vclip as x < -1 ? -1 : x > 1 ? 1 : x, so NaN passes through and +-inf clip to +-1.  A NaN
 *             comes out as the device's canonical NaN (its payload is not kept).
 */
#ifndef FLUIDAUDIO_B200_LUXTTS_H
#define FLUIDAUDIO_B200_LUXTTS_H

#include "fluidaudio_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define FA_LUXTTS_FEAT_DIM 100          /* LuxTtsConstants.featDim */
#define FA_LUXTTS_MAX_FRAMES 1024       /* LuxTtsConstants.maxFrames */
#define FA_LUXTTS_MAX_TOKENS 256        /* LuxTtsConstants.maxTokens */
#define FA_LUXTTS_MAX_PROMPT 120000     /* Int(maxPromptSeconds * melSampleRate) */
#define FA_LUXTTS_NUM_STEPS 4           /* LuxTtsConstants.numSteps */
#define FA_LUXTTS_HOP_48K 512           /* LuxTtsConstants.hop48k */
#define FA_LUXTTS_SAMPLE_RATE 48000     /* LuxTtsConstants.outputSampleRate */

/* Reason codes of a refused request, in the order synthesize's guards and LuxTtsError throw them. */
enum {
    FA_LUXTTS_OK = 0,
    FA_LUXTTS_NO_PROMPT_TOKENS = 1,       /* promptTokenIds is empty */
    FA_LUXTTS_NO_TEXT_TOKENS = 2,         /* textTokenIds is empty */
    FA_LUXTTS_NO_PROMPT_SAMPLES = 3,      /* promptAudio24k is empty */
    FA_LUXTTS_BAD_SPEED = 4,              /* !(speed > 0): 0, negative or NaN */
    FA_LUXTTS_SILENT_PROMPT = 5,          /* !(rms > 0), reported by fa_luxtts_begin only */
    FA_LUXTTS_PROMPT_TOO_SHORT = 6,       /* no mel frame: fewer than 128 samples */
    FA_LUXTTS_TOO_MANY_TOKENS = 7,        /* tokenCount + 1 > 256 */
    FA_LUXTTS_FEATURES_TOO_LONG = 8,      /* featuresLength > 1024, or where Swift's Int(...) would trap */
    FA_LUXTTS_TOO_FEW_FRAMES = 9,         /* genFrames < 2 */
    FA_LUXTTS_NO_BUCKET = 10,             /* no vocoder bucket in {282, 555} holds genFrames */
    FA_LUXTTS_DEGENERATE_DURATION = 11    /* featuresLength / tokenCount < 1 */
};

typedef struct {
    int32_t reason;           /* FA_LUXTTS_*; the fields below are set when it is FA_LUXTTS_OK (the first four whenever
                                 they were reached) */
    int32_t prompt_samples;   /* the prompt after the 120 000-sample cap */
    int32_t prompt_frames;    /* (prompt_samples + 128) / 256 */
    int32_t token_count;      /* prompt + text tokens */
    int32_t features_length;  /* prompt_frames + Int((Double(P) / Double(pt) * Double(tt) / Double(speed)).rounded(.up)) */
    int32_t gen_frames;       /* features_length - prompt_frames */
    int32_t bucket;           /* the first of 282, 555 that is >= gen_frames */
    int32_t boosted;          /* fa_luxtts_begin: rms < 0.1f, so the prompt was gained and the output is scaled back */
    float prompt_rms;         /* fa_luxtts_begin: sqrtf of the mean square */
    int32_t step;             /* fa_luxtts_request_state: FmDecoder steps applied, 0 .. 4 */
} fa_luxtts_plan_info;

/* The request geometry of synthesize, on the host.  featuresLength is evaluated in float64 in Swift's left-to-right
 * order, then rounded up; where Swift's Int(...) or the sum with prompt_frames would trap (an infinite or too large
 * value, reachable with a tiny speed) the request is refused as FA_LUXTTS_FEATURES_TOO_LONG.  Negative counts are
 * FA_STATUS_INVALID_ARGUMENT.  No launch. */
fa_status fa_luxtts_plan(int64_t prompt_samples, int32_t prompt_token_count, int32_t text_token_count, float speed,
                         fa_luxtts_plan_info *plan);

typedef struct fa_luxtts fa_luxtts;   /* one handle per stream of calls; not thread-safe */
fa_status fa_luxtts_create(fa_luxtts **out);
void fa_luxtts_destroy(fa_luxtts *h);

/* Opens `count` requests.  Request i's 24 kHz prompt is prompt[offsets[i] .. offsets[i+1]) (offsets non-decreasing
 * from offsets[0] >= 0), with prompt_tokens[i] / text_tokens[i] tokens, speeds[i] and seeds[i].  Every request is
 * planned and its mean square computed, then the call synchronises.  If any request is refused, reasons[i] holds each
 * request's code, the call returns FA_STATUS_INVALID_ARGUMENT and opens nothing.  Otherwise reasons[i] = 0, ids[i] and
 * plans[i] are set, and:
 *   speech_condition [count x 1024 x 100]  mel(gained prompt) x 0.1f for frames < prompt_frames, zeros after
 *   padding_mask     [count x 1024]        1.0f from features_length on, 0.0f before
 *   each slot                              the noise x0 for elements < features_length x 100, zeros after
 * 4 launches: RMS; gain into scratch; the mel batch; epilogue and noise. */
fa_status fa_luxtts_begin(fa_luxtts *h, int32_t count, const float *prompt, const int64_t *offsets,
                          const int32_t *prompt_tokens, const int32_t *text_tokens, const float *speeds,
                          const uint64_t *seeds, int32_t *reasons, int32_t *ids, fa_luxtts_plan_info *plans,
                          float *speech_condition, float *padding_mask);
fa_status fa_luxtts_begin_device(fa_luxtts *h, int32_t count, const float *d_prompt, const int64_t *offsets,
                                 const int32_t *prompt_tokens, const int32_t *text_tokens, const float *speeds,
                                 const uint64_t *seeds, int32_t *reasons, int32_t *ids, fa_luxtts_plan_info *plans,
                                 float *d_speech_condition, float *d_padding_mask);

/* text_condition [count x 1024 x 100]: row f < features_length is token_embeds row tokensIndex[f] of request i, zeros
 * after.  Request i's embeds start at token_embeds + i * request_stride, row r at + r * row_stride (row_stride >= 100,
 * request_stride >= (token_count + 1) * row_stride for every request named), rows 0 .. token_count are read.  Any step.
 * 1 launch. */
fa_status fa_luxtts_text_condition(fa_luxtts *h, int32_t count, const int32_t *ids, const float *token_embeds,
                                   int64_t row_stride, int64_t request_stride, float *text_condition);
fa_status fa_luxtts_text_condition_device(fa_luxtts *h, int32_t count, const int32_t *ids, const float *d_token_embeds,
                                          int64_t row_stride, int64_t request_stride, float *d_text_condition);

/* x [count x 1024 x 100] (the slot) and t [count] = Float(timeSteps[step]).  Requests at step 0 .. 3.  d_x must be
 * 16-byte aligned.  1 launch. */
fa_status fa_luxtts_model_inputs(fa_luxtts *h, int32_t count, const int32_t *ids, float *x, float *t);
fa_status fa_luxtts_model_inputs_device(fa_luxtts *h, int32_t count, const int32_t *ids, float *d_x, float *d_t);

/* One anchor-Euler update of each request's slot with the FmDecoder's v (rows 0 .. features_length - 1 of request i at
 * v + i * request_stride + row * row_stride, row_stride >= 100, request_stride >= features_length * row_stride), then
 * the step advances.  Requests at step 0 .. 3, which may differ within a call.  1 launch. */
fa_status fa_luxtts_advance(fa_luxtts *h, int32_t count, const int32_t *ids, const float *v, int64_t row_stride,
                            int64_t request_stride);
fa_status fa_luxtts_advance_device(fa_luxtts *h, int32_t count, const int32_t *ids, const float *d_v,
                                   int64_t row_stride, int64_t request_stride);

/* mel [count x 100 x bucket]: x[(prompt_frames + f) * 100 + m] * 10.0f for f < gen_frames, logf(1e-7f) after.
 * Requests at step 4 whose bucket is `bucket`.  1 launch (a shared-memory tile transpose). */
fa_status fa_luxtts_vocoder_input(fa_luxtts *h, int32_t count, const int32_t *ids, int32_t bucket, float *mel);
fa_status fa_luxtts_vocoder_input_device(fa_luxtts *h, int32_t count, const int32_t *ids, int32_t bucket, float *d_mel);

/* Request i's vocoder output is audio[i * row_stride .. + row_length) (row_length <= row_stride).  It keeps
 * lengths[i] = min((gen_frames - 1) * 512, row_length) samples, clips them to [-1, 1] and, for a boosted prompt,
 * multiplies them by prompt_rms / 0.1f (float32).  They are packed in request order into samples; *total is their sum.
 * When *total > capacity the call returns FA_STATUS_OUTPUT_TOO_SMALL with lengths and *total set, writes no sample and
 * closes nothing.  Otherwise every request is closed.  Requests at step 4.  1 launch (none when *total is 0). */
fa_status fa_luxtts_finish(fa_luxtts *h, int32_t count, const int32_t *ids, const float *audio, int64_t row_stride,
                           int64_t row_length, float *samples, size_t capacity, int64_t *lengths, int64_t *total);
fa_status fa_luxtts_finish_device(fa_luxtts *h, int32_t count, const int32_t *ids, const float *d_audio,
                                  int64_t row_stride, int64_t row_length, float *d_samples, size_t capacity,
                                  int64_t *lengths, int64_t *total);

/* Drops a request without finishing it. */
fa_status fa_luxtts_close(fa_luxtts *h, int32_t id);
/* The request's plan (with its step) and, when x is not NULL, its slot [1024 x 100].  Synchronises. */
fa_status fa_luxtts_request_state(fa_luxtts *h, int32_t id, fa_luxtts_plan_info *plan, float *x);

#ifdef __cplusplus
}
#endif

#endif /* FLUIDAUDIO_B200_LUXTTS_H */
