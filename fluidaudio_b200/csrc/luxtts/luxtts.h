// The host side of LuxTTS synthesis (luxtts_kernels.cu) behind the C ABI (luxtts_abi.cu): the request set.
#pragma once

#include "../mel_plan.h"
#include "../session_table.h"
#include "luxtts_core.cuh"

namespace fa {
namespace luxtts {

// int32 fields of a slot's meta row, written by begin and read by the later kernels: the request's geometry, whether
// its prompt was boosted and the bits of its RMS.  The step travels in each call's descriptors.
enum : int { kPromptFrames = 0, kFeatures = 1, kGen = 2, kTokens = 3, kBoosted = 4, kRmsBits = 5, kMetaFields = 8 };

struct Mirror {
    Plan plan;
    float rms = 0.0f;
    bool boosted = false;
    int step = 0;
};

struct BeginArgs {
    int count;
    const float *prompt;
    const int64_t *offsets;
    const int32_t *prompt_tokens, *text_tokens;
    const float *speeds;
    const uint64_t *seeds;
    int32_t *reasons, *ids;
    Mirror *plans;   // the opened requests' mirrors
    float *speech_condition, *padding_mask;
};

class RequestSet {
  public:
    int init();
    int begin(const BeginArgs &a, bool device);
    int text_condition(int count, const int *ids, const float *embeds, long long row_stride, long long request_stride,
                       bool device, float *out);
    int model_inputs(int count, const int *ids, bool device, float *x, float *t);
    int advance(int count, const int *ids, const float *v, long long row_stride, long long request_stride, bool device);
    int vocoder_input(int count, const int *ids, int bucket, bool device, float *mel);
    int finish(int count, const int *ids, const float *audio, long long row_stride, long long row_length, bool device,
               float *samples, long long capacity, int64_t *lengths, int64_t *total);
    int close(int id);
    int state(int id, Mirror *m, float *x);

  private:
    int check(int count, const int *ids, const char *where, int min_step, int max_step) const;
    int open_all(int count, const Mirror *next, int32_t *ids);

    Stream stream;   // declared first, so destroyed last
    mel::MelPlan mel;
    SessionTable<Mirror> table;
    DeviceBuffer<float> d_x;      // [slots x 1024 x 100]
    DeviceBuffer<int> d_meta;     // [slots x kMetaFields]
    UploadStage<> desc;           // the call's per-request descriptors
    DeviceBuffer<> d_io;          // device twins of a host-buffer call's arrays
    DeviceBuffer<> d_scratch;     // begin: the gained prompts, their mel and the RMS
    PinnedBuffer<float> h_rms;    // begin: the RMS read back for the silent-prompt check
};

} // namespace luxtts
} // namespace fa
