// The host side of offline Sortformer windows (offline_sortformer_kernels.cu) behind the C ABI
// (offline_sortformer_abi.cu): the two data-taking calls on a leased call context.  Arguments arrive checked, with
// the overlap clamped.
#pragma once

#include "../call_context.h"
#include "offline_sortformer_core.cuh"

namespace fa {
namespace offline_sortformer {

int model_inputs(CallContext &C, int overlap, int count, const float *mel, const int64_t *mel_offsets,
                 const int64_t *mel_frames, long long windows, bool device, float *model_mel, int32_t *mel_length);
int stitch(CallContext &C, int overlap, int count, const int64_t *mel_frames, const float *speaker_preds,
           long long windows, long long rows, bool device, float *predictions, int32_t *mappings);

} // namespace offline_sortformer
} // namespace fa
