// C ABI of StyleTTS2 synthesis glue (declared in include/fluidaudio_b200_styletts2.h) over styletts2_kernels.cu.  Every
// argument and request is checked here before any copy or launch; every entry point returns through guard()
// (c_abi.h), and the data-taking calls lease the pooled call context (call_context.h).
#include "../../../include/fluidaudio_b200_styletts2.h"
#include "../c_abi.h"
#include "styletts2.h"

// The family's entry points: C linkage, exported, returning the main header's fa_status.  The library-wide guard scan
// (tests/test_abi_errors.py) keeps a closed list of family headers; tests/test_styletts2_abi.py holds every entry
// point spelled this way to the same rule: one statement, `return guard(__func__, ...)`.
#define FA_STYLETTS2_API FA_API fa_status

using namespace fa;
using namespace fa::styletts2;

namespace {

int sampler_call(int count, const int32_t *ids, const int64_t *offsets, const uint64_t *seeds, int bucket,
                 int32_t *tokens, int32_t *mask, float *noise, int32_t *reasons, bool device) {
    const char *where = device ? "fa_styletts2_sampler_inputs_device" : "fa_styletts2_sampler_inputs";
    if (count < 0) return refuse("%s: count %d < 0", where, count);
    if (bucket != kDefaultTokens && bucket != 64 && bucket != 128 && bucket != kMaxTokens)
        return refuse("%s: bucket %d is not 57, 64, 128 or 256", where, bucket);
    if (count == 0) return FA_STATUS_OK;
    if (!offsets || !seeds || !reasons || !tokens || !mask || !noise)
        return refuse("%s: offsets, seeds, reasons, tokens, attention_mask and noise must be non-null", where);
    if (offsets[0] < 0) return refuse("%s: offsets[0] is negative (%lld)", where, (long long)offsets[0]);
    for (int i = 0; i < count; ++i)
        if (offsets[i + 1] < offsets[i] || offsets[i + 1] > (1LL << 62))
            return refuse("%s: offsets decrease at %d or pass 2^62", where, i);
    int refused = -1, other = -1;
    for (int i = 0; i < count; ++i) {
        const long long n = offsets[i + 1] - offsets[i];
        int r = kOk;
        const int b = n > kMaxTokens ? (r = kNoBucket, 0) : bucket_for((int)n, &r);
        reasons[i] = r;
        if (r != kOk && refused < 0) refused = i;
        if (r == kOk && b != bucket && other < 0) other = i;
    }
    if (refused >= 0)
        return refuse("%s: request %d is refused with reason %d (see reasons)", where, refused, reasons[refused]);
    if (other >= 0)
        return refuse("%s: request %d has %lld tokens, outside bucket %d", where, other,
                      (long long)(offsets[other + 1] - offsets[other]), bucket);
    if (!ids) return refuse("%s: token_ids is NULL", where);
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) {
        return sampler_inputs(C, count, ids, offsets, seeds, bucket, device, tokens, mask, noise);
    });
}

int style_call(int count, const float *s_pred, const float *ref_s, const float *alphas, const float *betas,
               float *ref, float *s, bool device) {
    const char *where = device ? "fa_styletts2_style_device" : "fa_styletts2_style";
    if (count < 0) return refuse("%s: count %d < 0", where, count);
    if (count == 0) return FA_STATUS_OK;
    if (!s_pred || !ref_s || !alphas || !betas || !ref || !s)
        return refuse("%s: s_pred, ref_s, alphas, betas, ref and s must be non-null", where);
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) { return style(C, count, s_pred, ref_s, alphas, betas, device, ref, s); });
}

int align_call(const AlignArgs &a, bool device) {
    const char *where = device ? "fa_styletts2_align_device" : "fa_styletts2_align";
    if (a.count < 0) return refuse("%s: count %d < 0", where, a.count);
    if (a.count == 0) return FA_STATUS_OK;
    if (!a.token_counts || !a.logits || !a.d || !a.t_en || !a.en || !a.asr || !a.frames || !a.reasons)
        return refuse("%s: token_counts, logits, d, t_en, en, asr, frames and reasons must be non-null", where);
    if (a.channels < 1 || a.channels > (1 << 24)) return refuse("%s: logit_channels %d is outside 1 .. 2^24", where, a.channels);
    if (a.d_channels < 1 || a.d_channels > (1 << 20) || a.t_channels < 1 || a.t_channels > (1 << 20))
        return refuse("%s: d_channels %d and t_en_channels %d must be 1 .. 2^20", where, a.d_channels, a.t_channels);
    if (a.frame_stride < 1 || a.frame_stride > (1LL << 22))
        return refuse("%s: frame_stride %lld is outside 1 .. 2^22", where, a.frame_stride);
    if (a.logit_row < a.channels || a.logit_row > (1LL << 40))
        return refuse("%s: logit_row_stride %lld < logit_channels %d", where, a.logit_row, a.channels);
    if (a.d_row < a.d_channels || a.d_row > (1LL << 40))
        return refuse("%s: d_row_stride %lld < d_channels %d", where, a.d_row, a.d_channels);
    for (int i = 0; i < a.count; ++i) {
        const long long n = a.token_counts[i];
        if (n < 1 || n > kMaxTokens) return refuse("%s: request %d has %lld tokens, not 1 .. 256", where, i, n);
        if (a.logit_request < n * a.logit_row || a.logit_request > (1LL << 50))
            return refuse("%s: logit_request_stride %lld does not hold request %d's %lld rows", where, a.logit_request,
                          i, n);
        if (a.d_request < n * a.d_row || a.d_request > (1LL << 50))
            return refuse("%s: d_request_stride %lld does not hold request %d's %lld rows", where, a.d_request, i, n);
        if (a.t_row < n || a.t_row > (1LL << 40) || a.t_request < a.t_channels * a.t_row || a.t_request > (1LL << 50))
            return refuse("%s: t_en_row_stride %lld / t_en_request_stride %lld do not hold request %d's %d x %lld",
                          where, a.t_row, a.t_request, i, a.t_channels, n);
    }
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) { return align(C, a, device, where); });
}

} // namespace

FA_STYLETTS2_API fa_styletts2_plan(int32_t token_count, int32_t *bucket, int32_t *reason) {
    return guard(__func__, [&]() -> int {
        if (!bucket || !reason) return refuse("fa_styletts2_plan: bucket or reason is NULL");
        if (token_count < 0) return refuse("fa_styletts2_plan: token_count %d < 0", token_count);
        int r = kOk;
        *bucket = bucket_for(token_count, &r);
        *reason = r;
        return FA_STATUS_OK;
    });
}

FA_STYLETTS2_API fa_styletts2_sampler_inputs(int32_t count, const int32_t *token_ids, const int64_t *offsets,
                                             const uint64_t *seeds, int32_t bucket, int32_t *tokens,
                                             int32_t *attention_mask, float *noise, int32_t *reasons) {
    return guard(__func__, [&] {
        return sampler_call(count, token_ids, offsets, seeds, bucket, tokens, attention_mask, noise, reasons, false);
    });
}

FA_STYLETTS2_API fa_styletts2_sampler_inputs_device(int32_t count, const int32_t *d_token_ids, const int64_t *offsets,
                                                    const uint64_t *seeds, int32_t bucket, int32_t *d_tokens,
                                                    int32_t *d_attention_mask, float *d_noise, int32_t *reasons) {
    return guard(__func__, [&] {
        return sampler_call(count, d_token_ids, offsets, seeds, bucket, d_tokens, d_attention_mask, d_noise, reasons,
                            true);
    });
}

FA_STYLETTS2_API fa_styletts2_style(int32_t count, const float *s_pred, const float *ref_s, const float *alphas,
                                    const float *betas, float *ref, float *s) {
    return guard(__func__, [&] { return style_call(count, s_pred, ref_s, alphas, betas, ref, s, false); });
}

FA_STYLETTS2_API fa_styletts2_style_device(int32_t count, const float *d_s_pred, const float *d_ref_s,
                                           const float *alphas, const float *betas, float *d_ref, float *d_s) {
    return guard(__func__, [&] { return style_call(count, d_s_pred, d_ref_s, alphas, betas, d_ref, d_s, true); });
}

FA_STYLETTS2_API fa_styletts2_align(int32_t count, const int32_t *token_counts, const float *logits,
                                    int32_t logit_channels, int64_t logit_row_stride, int64_t logit_request_stride,
                                    const float *d, int32_t d_channels, int64_t d_row_stride, int64_t d_request_stride,
                                    const float *t_en, int32_t t_en_channels, int64_t t_en_row_stride,
                                    int64_t t_en_request_stride, int64_t frame_stride, float *en, float *asr,
                                    int64_t *frames, int32_t *durations, int32_t *reasons) {
    return guard(__func__, [&] {
        return align_call(AlignArgs{count, token_counts, logits, logit_channels, logit_row_stride, logit_request_stride,
                                    d, d_channels, d_row_stride, d_request_stride, t_en, t_en_channels,
                                    t_en_row_stride, t_en_request_stride, frame_stride, en, asr, frames, durations,
                                    reasons},
                          false);
    });
}

FA_STYLETTS2_API fa_styletts2_align_device(int32_t count, const int32_t *token_counts, const float *d_logits,
                                           int32_t logit_channels, int64_t logit_row_stride,
                                           int64_t logit_request_stride, const float *d_d, int32_t d_channels,
                                           int64_t d_row_stride, int64_t d_request_stride, const float *d_t_en,
                                           int32_t t_en_channels, int64_t t_en_row_stride,
                                           int64_t t_en_request_stride, int64_t frame_stride, float *d_en,
                                           float *d_asr, int64_t *frames, int32_t *durations, int32_t *reasons) {
    return guard(__func__, [&] {
        return align_call(AlignArgs{count, token_counts, d_logits, logit_channels, logit_row_stride,
                                    logit_request_stride, d_d, d_channels, d_row_stride, d_request_stride, d_t_en,
                                    t_en_channels, t_en_row_stride, t_en_request_stride, frame_stride, d_en, d_asr,
                                    frames, durations, reasons},
                          true);
    });
}
