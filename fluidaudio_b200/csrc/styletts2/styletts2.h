// The host side of StyleTTS2 synthesis glue (styletts2_kernels.cu) behind the C ABI (styletts2_abi.cu): the three
// data-taking calls on a leased call context.  Arguments arrive checked.
#pragma once

#include "../call_context.h"
#include "styletts2_core.cuh"

namespace fa {
namespace styletts2 {

struct AlignArgs {
    int count;
    const int32_t *token_counts;
    const float *logits;
    int channels;
    long long logit_row, logit_request;
    const float *d;
    int d_channels;
    long long d_row, d_request;
    const float *t_en;
    int t_channels;
    long long t_row, t_request;
    long long frame_stride;
    float *en, *asr;
    int64_t *frames;
    int32_t *durations, *reasons;
};

int sampler_inputs(CallContext &C, int count, const int32_t *token_ids, const int64_t *offsets, const uint64_t *seeds,
                   int bucket, bool device, int32_t *tokens, int32_t *mask, float *noise);
int style(CallContext &C, int count, const float *s_pred, const float *ref_s, const float *alphas, const float *betas,
          bool device, float *ref, float *s);
int align(CallContext &C, const AlignArgs &a, bool device, const char *where);

} // namespace styletts2
} // namespace fa
