// C ABI of the Sortformer streaming state (declared in include/fluidaudio_b200.h):
// SortformerStateUpdater.streamingUpdate for many sessions in HBM, sortformer_streams.cu and sortformer_kernels.cu.
// Every entry point that returns a status returns through guard() (c_abi.h).
#include "c_abi.h"
#include "sortformer_plan.h"

#include <algorithm>
#include <cstring>
#include <memory>

struct fa_sortformer {
    fa::sortformer::SortformerSet set;
};

using namespace fa;

static sortformer::Config sortformer_config_of(const fa_sortformer_config *c) {
    sortformer::Config s{};
    s.chunk_len = c->chunk_len;
    s.left_context = c->chunk_left_context;
    s.right_context = c->chunk_right_context;
    s.fifo_len = c->fifo_len;
    s.spkcache_len = c->spkcache_len;
    s.update_period = c->spkcache_update_period;
    s.sil_per_spk = c->spkcache_sil_frames_per_spk;
    s.silence_threshold = c->silence_threshold;
    s.pred_score_threshold = c->pred_score_threshold;
    s.scores_boost_latest = c->scores_boost_latest;
    s.strong_boost_rate = c->strong_boost_rate;
    s.weak_boost_rate = c->weak_boost_rate;
    s.min_pos_scores_rate = c->min_pos_scores_rate;
    return s;
}

FA_API fa_status fa_sortformer_default_config(fa_sortformer_config *cfg, int32_t preset) {
    return guard(__func__, [&]() -> int {
        if (!cfg) return FA_STATUS_INVALID_ARGUMENT;
        // SortformerTypes.swift:121-216: chunkLen, left, right context, fifoLen, spkcacheLen, update period
        static const int32_t presets[8][6] = {
            {6, 1, 7, 40, 188, 31},    {6, 1, 7, 40, 188, 31},   {6, 1, 7, 40, 188, 31},   {6, 1, 7, 188, 188, 144},
            {6, 1, 7, 188, 188, 144},  {340, 1, 40, 40, 188, 300}, {340, 1, 40, 40, 188, 300}, {25, 1, 7, 40, 188, 31},
        };
        if (preset < 0 || preset > 7) return refuse("fa_sortformer_default_config: unknown preset %d", preset);
        const int32_t *p = presets[preset];
        // the init's defaults (SortformerTypes.swift:219-236) and its clamps, as the static configs hold them:
        // highContext's period 300 becomes chunkLen = 340
        *cfg = fa_sortformer_config{p[0], p[1], p[2], p[3], p[4], p[5], 3, 0.2f, 0.25f, 0.05f, 0.75f, 1.5f, 0.5f};
        cfg->spkcache_update_period = std::max(std::min(p[5], p[3] + p[0]), p[0]);
        return FA_STATUS_OK;
    });
}

static void sortformer_config_out(const sortformer::Config &c, fa_sortformer_config *o) {
    *o = fa_sortformer_config{c.chunk_len, c.left_context, c.right_context, c.fifo_len, c.spkcache_len, c.update_period,
                              c.sil_per_spk, c.silence_threshold, c.pred_score_threshold, c.scores_boost_latest,
                              c.strong_boost_rate, c.weak_boost_rate, c.min_pos_scores_rate};
}

FA_API fa_status fa_sortformer_resolve_config(const fa_sortformer_config *cfg, int32_t max_core_frames,
                                              fa_sortformer_config *resolved, int32_t *resolved_max_core) {
    return guard(__func__, [&]() -> int {
        if (!cfg) return FA_STATUS_INVALID_ARGUMENT;
        sortformer::Config c;
        const int st = sortformer::resolve_config(sortformer_config_of(cfg), max_core_frames, c);
        if (st != FA_OK) return st;
        if (resolved) sortformer_config_out(c, resolved);
        if (resolved_max_core) *resolved_max_core = c.max_core;
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_sortformer_step(const fa_sortformer_config *cfg, int32_t max_core_frames, const int32_t *lengths_in,
                                    int32_t emb_length, int32_t pred_rows, int32_t left_context, int32_t right_context,
                                    int32_t *out) {
    return guard(__func__, [&]() -> int {
        if (!cfg || !lengths_in || !out) return FA_STATUS_INVALID_ARGUMENT;
        sortformer::Config c;
        int st = sortformer::resolve_config(sortformer_config_of(cfg), max_core_frames, c);
        if (st != FA_OK) return st;
        if (lengths_in[0] < 0 || lengths_in[0] > c.spkcache_len || lengths_in[1] < 0 || lengths_in[1] > c.fifo_len)
            return refuse("fa_sortformer_step: lengths (%d, %d) outside the state's bounds", lengths_in[0], lengths_in[1]);
        sortformer::Step s;
        st = sortformer::plan_step(c, lengths_in[0], lengths_in[1], lengths_in[2] != 0, emb_length, pred_rows,
                                   left_context, right_context, s);
        if (st != FA_OK) return st;
        const int32_t v[6] = {s.core, s.pop, s.compress, s.spkcache_after, s.fifo_after, s.has_preds_after};
        std::memcpy(out, v, sizeof(v));
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_sortformer_create(const fa_sortformer_config *cfg, int32_t max_core_frames, fa_sortformer **out) {
    return guard(__func__, [&]() -> int {
        if (!cfg || !out) return FA_STATUS_INVALID_ARGUMENT;
        *out = nullptr;
        sortformer::Config c;
        int st = sortformer::resolve_config(sortformer_config_of(cfg), max_core_frames, c);
        if (st != FA_OK) return st;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        std::unique_ptr<fa_sortformer> h(new fa_sortformer());
        st = h->set.init(c);
        if (st != FA_OK) return st;
        *out = h.release();
        return FA_STATUS_OK;
    });
}

FA_API void fa_sortformer_destroy(fa_sortformer *h) { delete h; }

FA_API fa_status fa_sortformer_open(fa_sortformer *h, int32_t *session) {
    return guard(__func__, [&]() -> int {
        if (!h || !session) return FA_STATUS_INVALID_ARGUMENT;
        int id = -1;
        const int st = h->set.open(&id);
        if (st == FA_OK) *session = id;
        return st;
    });
}

FA_API fa_status fa_sortformer_close(fa_sortformer *h, int32_t session) {
    return guard(__func__, [&]() -> int {
        if (!h) return FA_STATUS_INVALID_ARGUMENT;
        return h->set.close(session);
    });
}

static int sortformer_update(fa_sortformer *h, int32_t count, const int32_t *sessions, const float *embs,
                             int32_t emb_rows, const float *preds, int32_t pred_rows, const int32_t *emb_lengths,
                             const int32_t *left, const int32_t *right, bool device, float *confirmed,
                             size_t confirmed_len, float *tentative, size_t tentative_len, int64_t *confirmed_rows,
                             int64_t *tentative_rows) {
    if (!h) return FA_STATUS_INVALID_ARGUMENT;
    return h->set.update(count, sessions, embs, emb_rows, preds, pred_rows, emb_lengths, left, right, device, confirmed,
                         capacity(confirmed_len), tentative, capacity(tentative_len), confirmed_rows, tentative_rows);
}

FA_API fa_status fa_sortformer_update(fa_sortformer *h, int32_t count, const int32_t *sessions, const float *chunk_embs,
                                      int32_t emb_rows, const float *preds, int32_t pred_rows, const int32_t *emb_lengths,
                                      const int32_t *left_context, const int32_t *right_context, float *confirmed,
                                      size_t confirmed_len, float *tentative, size_t tentative_len,
                                      int64_t *confirmed_rows, int64_t *tentative_rows) {
    return guard(__func__, [&] {
        return sortformer_update(h, count, sessions, chunk_embs, emb_rows, preds, pred_rows, emb_lengths, left_context,
                                 right_context, false, confirmed, confirmed_len, tentative, tentative_len,
                                 confirmed_rows, tentative_rows);
    });
}

FA_API fa_status fa_sortformer_update_device(fa_sortformer *h, int32_t count, const int32_t *sessions,
                                             const float *d_chunk_embs, int32_t emb_rows, const float *d_preds,
                                             int32_t pred_rows, const int32_t *emb_lengths, const int32_t *left_context,
                                             const int32_t *right_context, float *d_confirmed, size_t confirmed_len,
                                             float *d_tentative, size_t tentative_len, int64_t *confirmed_rows,
                                             int64_t *tentative_rows) {
    return guard(__func__, [&] {
        return sortformer_update(h, count, sessions, d_chunk_embs, emb_rows, d_preds, pred_rows, emb_lengths,
                                 left_context, right_context, true, d_confirmed, confirmed_len, d_tentative,
                                 tentative_len, confirmed_rows, tentative_rows);
    });
}

static int sortformer_inputs(fa_sortformer *h, int32_t count, const int32_t *sessions, bool device, float *spkcache,
                             float *fifo, int32_t *spkcache_lengths, int32_t *fifo_lengths) {
    if (!h) return FA_STATUS_INVALID_ARGUMENT;
    return h->set.model_inputs(count, sessions, device, spkcache, fifo, spkcache_lengths, fifo_lengths);
}

FA_API fa_status fa_sortformer_model_inputs(fa_sortformer *h, int32_t count, const int32_t *sessions, float *spkcache,
                                            float *fifo, int32_t *spkcache_lengths, int32_t *fifo_lengths) {
    return guard(__func__, [&] {
        return sortformer_inputs(h, count, sessions, false, spkcache, fifo, spkcache_lengths, fifo_lengths);
    });
}

FA_API fa_status fa_sortformer_model_inputs_device(fa_sortformer *h, int32_t count, const int32_t *sessions,
                                                   float *d_spkcache, float *d_fifo, int32_t *spkcache_lengths,
                                                   int32_t *fifo_lengths) {
    return guard(__func__, [&] {
        return sortformer_inputs(h, count, sessions, true, d_spkcache, d_fifo, spkcache_lengths, fifo_lengths);
    });
}

FA_API fa_status fa_sortformer_session_state(fa_sortformer *h, int32_t session, fa_sortformer_session_info *info,
                                             float *spkcache, float *spkcache_preds, float *fifo, float *fifo_preds,
                                             float *mean_silence) {
    return guard(__func__, [&]() -> int {
        if (!h || !info) return FA_STATUS_INVALID_ARGUMENT;
        sortformer::SessionInfo s;
        const int st = h->set.state(session, &s, spkcache, spkcache_preds, fifo, fifo_preds, mean_silence);
        if (st != FA_OK) return st;
        *info = fa_sortformer_session_info{s.spkcache_length, s.fifo_length, s.has_spkcache_preds, s.has_fifo_preds,
                                           s.chunks,          s.silence_frames};
        return FA_STATUS_OK;
    });
}
