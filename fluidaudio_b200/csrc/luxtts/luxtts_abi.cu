// C ABI of LuxTTS synthesis (declared in include/fluidaudio_b200_luxtts.h) over luxtts_kernels.cu.  Every argument is
// checked here or in the request set before any copy or launch; every entry point that returns a status returns
// through guard() (c_abi.h).
#include "../../../include/fluidaudio_b200_luxtts.h"
#include "../c_abi.h"
#include "luxtts.h"

#include <memory>
#include <vector>

// The family's status-returning entry points: C linkage, exported, returning the main header's fa_status.  The
// library-wide guard scan (tests/test_abi_errors.py) keeps a closed list of family headers; tests/test_luxtts_abi.py
// holds every entry point spelled this way to the same rule: one statement, `return guard(__func__, ...)`.
#define FA_LUXTTS_API FA_API fa_status

struct fa_luxtts {
    fa::luxtts::RequestSet set;
};

using namespace fa;
using namespace fa::luxtts;

namespace {

fa_luxtts_plan_info info_of(const Mirror &m) {
    const Plan &p = m.plan;
    return fa_luxtts_plan_info{p.reason,     p.prompt_samples, p.prompt_frames,  p.token_count, p.features_length,
                               p.gen_frames, p.bucket,         m.boosted ? 1 : 0, m.rms,        m.step};
}

int begin(fa_luxtts *h, int32_t count, const float *prompt, const int64_t *offsets, const int32_t *prompt_tokens,
          const int32_t *text_tokens, const float *speeds, const uint64_t *seeds, int32_t *reasons, int32_t *ids,
          fa_luxtts_plan_info *plans, float *speech_condition, float *padding_mask, bool device) {
    if (!h) return refuse("%s: h is NULL", device ? "fa_luxtts_begin_device" : "fa_luxtts_begin");
    std::vector<Mirror> mirrors(count > 0 ? (size_t)count : 0);
    const BeginArgs a{count,   prompt, offsets, prompt_tokens,  text_tokens, speeds,
                      seeds,   reasons, ids,    mirrors.data(), speech_condition, padding_mask};
    const int st = h->set.begin(a, device);
    if (st == FA_OK && plans)
        for (int i = 0; i < count; ++i) plans[i] = info_of(mirrors[(size_t)i]);
    return st;
}

} // namespace

FA_LUXTTS_API fa_luxtts_plan(int64_t prompt_samples, int32_t prompt_token_count, int32_t text_token_count,
                             float speed, fa_luxtts_plan_info *plan) {
    return guard(__func__, [&]() -> int {
        if (!plan) return refuse("fa_luxtts_plan: plan is NULL");
        if (prompt_samples < 0 || prompt_token_count < 0 || text_token_count < 0)
            return refuse("fa_luxtts_plan: negative count (%lld samples, %d prompt tokens, %d text tokens)",
                          (long long)prompt_samples, prompt_token_count, text_token_count);
        Mirror m;
        m.plan = plan_request(prompt_samples, prompt_token_count, text_token_count, speed);
        *plan = info_of(m);
        return FA_STATUS_OK;
    });
}

FA_LUXTTS_API fa_luxtts_create(fa_luxtts **out) {
    return guard(__func__, [&]() -> int {
        if (!out) return refuse("fa_luxtts_create: out is NULL");
        *out = nullptr;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        std::unique_ptr<fa_luxtts> h(new fa_luxtts());
        const int st = h->set.init();
        if (st != FA_OK) return st;
        *out = h.release();
        return FA_STATUS_OK;
    });
}

FA_API void fa_luxtts_destroy(fa_luxtts *h) { delete h; }

FA_LUXTTS_API fa_luxtts_begin(fa_luxtts *h, int32_t count, const float *prompt, const int64_t *offsets,
                              const int32_t *prompt_tokens, const int32_t *text_tokens, const float *speeds,
                              const uint64_t *seeds, int32_t *reasons, int32_t *ids, fa_luxtts_plan_info *plans,
                              float *speech_condition, float *padding_mask) {
    return guard(__func__, [&] {
        return begin(h, count, prompt, offsets, prompt_tokens, text_tokens, speeds, seeds, reasons, ids, plans,
                     speech_condition, padding_mask, false);
    });
}

FA_LUXTTS_API fa_luxtts_begin_device(fa_luxtts *h, int32_t count, const float *d_prompt, const int64_t *offsets,
                                     const int32_t *prompt_tokens, const int32_t *text_tokens, const float *speeds,
                                     const uint64_t *seeds, int32_t *reasons, int32_t *ids,
                                     fa_luxtts_plan_info *plans, float *d_speech_condition, float *d_padding_mask) {
    return guard(__func__, [&] {
        return begin(h, count, d_prompt, offsets, prompt_tokens, text_tokens, speeds, seeds, reasons, ids, plans,
                     d_speech_condition, d_padding_mask, true);
    });
}

FA_LUXTTS_API fa_luxtts_text_condition(fa_luxtts *h, int32_t count, const int32_t *ids, const float *token_embeds,
                                       int64_t row_stride, int64_t request_stride, float *text_condition) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.text_condition(count, ids, token_embeds, row_stride, request_stride, false, text_condition)
                 : refuse("fa_luxtts_text_condition: h is NULL");
    });
}

FA_LUXTTS_API fa_luxtts_text_condition_device(fa_luxtts *h, int32_t count, const int32_t *ids,
                                              const float *d_token_embeds, int64_t row_stride,
                                              int64_t request_stride, float *d_text_condition) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.text_condition(count, ids, d_token_embeds, row_stride, request_stride, true, d_text_condition)
                 : refuse("fa_luxtts_text_condition_device: h is NULL");
    });
}

FA_LUXTTS_API fa_luxtts_model_inputs(fa_luxtts *h, int32_t count, const int32_t *ids, float *x, float *t) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.model_inputs(count, ids, false, x, t) : refuse("fa_luxtts_model_inputs: h is NULL");
    });
}

FA_LUXTTS_API fa_luxtts_model_inputs_device(fa_luxtts *h, int32_t count, const int32_t *ids, float *d_x,
                                            float *d_t) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.model_inputs(count, ids, true, d_x, d_t) : refuse("fa_luxtts_model_inputs_device: h is NULL");
    });
}

FA_LUXTTS_API fa_luxtts_advance(fa_luxtts *h, int32_t count, const int32_t *ids, const float *v, int64_t row_stride,
                                int64_t request_stride) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.advance(count, ids, v, row_stride, request_stride, false)
                 : refuse("fa_luxtts_advance: h is NULL");
    });
}

FA_LUXTTS_API fa_luxtts_advance_device(fa_luxtts *h, int32_t count, const int32_t *ids, const float *d_v,
                                       int64_t row_stride, int64_t request_stride) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.advance(count, ids, d_v, row_stride, request_stride, true)
                 : refuse("fa_luxtts_advance_device: h is NULL");
    });
}

FA_LUXTTS_API fa_luxtts_vocoder_input(fa_luxtts *h, int32_t count, const int32_t *ids, int32_t bucket, float *mel) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.vocoder_input(count, ids, bucket, false, mel) : refuse("fa_luxtts_vocoder_input: h is NULL");
    });
}

FA_LUXTTS_API fa_luxtts_vocoder_input_device(fa_luxtts *h, int32_t count, const int32_t *ids, int32_t bucket,
                                             float *d_mel) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.vocoder_input(count, ids, bucket, true, d_mel)
                 : refuse("fa_luxtts_vocoder_input_device: h is NULL");
    });
}

FA_LUXTTS_API fa_luxtts_finish(fa_luxtts *h, int32_t count, const int32_t *ids, const float *audio,
                               int64_t row_stride, int64_t row_length, float *samples, size_t capacity,
                               int64_t *lengths, int64_t *total) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.finish(count, ids, audio, row_stride, row_length, false, samples, fa::capacity(capacity),
                                 lengths, total)
                 : refuse("fa_luxtts_finish: h is NULL");
    });
}

FA_LUXTTS_API fa_luxtts_finish_device(fa_luxtts *h, int32_t count, const int32_t *ids, const float *d_audio,
                                      int64_t row_stride, int64_t row_length, float *d_samples, size_t capacity,
                                      int64_t *lengths, int64_t *total) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.finish(count, ids, d_audio, row_stride, row_length, true, d_samples, fa::capacity(capacity),
                                 lengths, total)
                 : refuse("fa_luxtts_finish_device: h is NULL");
    });
}

FA_LUXTTS_API fa_luxtts_close(fa_luxtts *h, int32_t id) {
    return guard(__func__, [&]() -> int { return h ? h->set.close(id) : refuse("fa_luxtts_close: h is NULL"); });
}

FA_LUXTTS_API fa_luxtts_request_state(fa_luxtts *h, int32_t id, fa_luxtts_plan_info *plan, float *x) {
    return guard(__func__, [&]() -> int {
        if (!h || !plan) return refuse("fa_luxtts_request_state: h or plan is NULL");
        Mirror m;
        const int st = h->set.state(id, &m, x);
        if (st == FA_OK) *plan = info_of(m);
        return st;
    });
}
