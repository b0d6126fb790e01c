// C ABI of the LS-EEND feature streams (declared in include/fluidaudio_b200_lseend.h): LSEENDFeatureProvider
// (LSEENDPreprocessor.swift:46-384) for many live sessions in HBM, lseend_plan.h and lseend_streams.cu.  Every entry point
// that returns a status returns through guard() (c_abi.h), as in every family's C ABI file.
#include "../../../include/fluidaudio_b200_lseend.h"
#include "c_abi.h"
#include "lseend_streams.h"

#include <cstring>
#include <memory>

struct fa_lseend_stream {
    fa::lseend::StreamSet set;
};

using namespace fa;

static lseend::Config lseend_config_of(const fa_lseend_stream_config *c) {
    return lseend::Config{c->sample_rate, c->n_mels,      c->hop_length, c->win_length, c->context_size,
                          c->subsampling, c->chunk_size, c->conv_delay, c->precision};
}

FA_API fa_status fa_lseend_stream_resolve(const fa_lseend_stream_config *cfg, fa_lseend_stream_sizes *sizes) {
    return guard(__func__, [&]() -> int {
        if (!cfg || !sizes) return FA_STATUS_INVALID_ARGUMENT;
        lseend::Sizes s;
        const int st = lseend::resolve(lseend_config_of(cfg), s);
        if (st != FA_OK) return st;
        *sizes = fa_lseend_stream_sizes{s.n_fft,         s.mel_frames,  s.chunk_mels,    s.mel_context,
                                        s.chunk_samples, s.audio_left,  s.audio_context, s.flush_samples,
                                        s.mask_length,   s.audio_capacity};
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_lseend_stream_create(const fa_lseend_stream_config *cfg, fa_lseend_stream **out) {
    return guard(__func__, [&]() -> int {
        if (!cfg || !out) return FA_STATUS_INVALID_ARGUMENT;
        *out = nullptr;
        lseend::Sizes s;
        int st = lseend::resolve(lseend_config_of(cfg), s);
        if (st != FA_OK) return st;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        std::unique_ptr<fa_lseend_stream> h(new fa_lseend_stream());
        st = h->set.init(lseend_config_of(cfg));
        if (st != FA_OK) return st;
        *out = h.release();
        return FA_STATUS_OK;
    });
}

FA_API void fa_lseend_stream_destroy(fa_lseend_stream *h) { delete h; }

FA_API fa_status fa_lseend_stream_open(fa_lseend_stream *h, int32_t *session) {
    return guard(__func__, [&]() -> int {
        if (!h || !session) return FA_STATUS_INVALID_ARGUMENT;
        int id = -1;
        const int st = h->set.open(&id);
        if (st == FA_OK) *session = id;
        return st;
    });
}

FA_API fa_status fa_lseend_stream_close(fa_lseend_stream *h, int32_t session) {
    return guard(__func__, [&]() -> int {
        if (!h) return FA_STATUS_INVALID_ARGUMENT;
        return h->set.close(session);
    });
}

FA_API int64_t fa_lseend_stream_chunks(const fa_lseend_stream *h, int32_t session, int64_t new_samples, int32_t drain) {
    const long long chunks = h ? h->set.chunks(session, new_samples, drain != 0) : -1;
    if (chunks < 0)
        fa::set_error("fa_lseend_stream_chunks: h is NULL, session %d is not open or new_samples is outside 0 .. 2^40",
                      session);
    return chunks;
}

static int lseend_stream_push(fa_lseend_stream *h, int32_t count, const int32_t *sessions, const float *audio,
                              const int64_t *offsets, const int32_t *drain, bool device, float *features,
                              size_t features_len, float *masks, size_t masks_len, int32_t *warmup, size_t warmup_len,
                              int64_t *chunks) {
    if (!h) return FA_STATUS_INVALID_ARGUMENT;
    return h->set.push(count, sessions, audio, offsets, drain, device, features, capacity(features_len), masks,
                       capacity(masks_len), warmup, capacity(warmup_len), chunks);
}

FA_API fa_status fa_lseend_stream_push(fa_lseend_stream *h, int32_t count, const int32_t *sessions, const float *audio,
                                       const int64_t *offsets, const int32_t *drain, float *features,
                                       size_t features_len, float *masks, size_t masks_len, int32_t *warmup,
                                       size_t warmup_len, int64_t *chunks) {
    return guard(__func__, [&] {
        return lseend_stream_push(h, count, sessions, audio, offsets, drain, false, features, features_len, masks,
                                  masks_len, warmup, warmup_len, chunks);
    });
}

FA_API fa_status fa_lseend_stream_push_device(fa_lseend_stream *h, int32_t count, const int32_t *sessions,
                                              const float *d_audio, const int64_t *offsets, const int32_t *drain,
                                              float *d_features, size_t features_len, float *d_masks, size_t masks_len,
                                              int32_t *d_warmup, size_t warmup_len, int64_t *chunks) {
    return guard(__func__, [&] {
        return lseend_stream_push(h, count, sessions, d_audio, offsets, drain, true, d_features, features_len, d_masks,
                                  masks_len, d_warmup, warmup_len, chunks);
    });
}

FA_API fa_status fa_lseend_stream_snapshot(fa_lseend_stream *h, int32_t count, const int32_t *sessions) {
    return guard(__func__, [&]() -> int { return h ? h->set.snapshot(count, sessions) : FA_STATUS_INVALID_ARGUMENT; });
}

FA_API fa_status fa_lseend_stream_rollback(fa_lseend_stream *h, int32_t count, const int32_t *sessions) {
    return guard(__func__, [&]() -> int { return h ? h->set.rollback(count, sessions) : FA_STATUS_INVALID_ARGUMENT; });
}

FA_API fa_status fa_lseend_stream_reset(fa_lseend_stream *h, int32_t count, const int32_t *sessions) {
    return guard(__func__, [&]() -> int { return h ? h->set.reset(count, sessions) : FA_STATUS_INVALID_ARGUMENT; });
}

FA_API fa_status fa_lseend_stream_session_state(fa_lseend_stream *h, int32_t session,
                                                fa_lseend_stream_session_info *info, float *audio, float *mel,
                                                float *cmn_mean) {
    return guard(__func__, [&]() -> int {
        if (!h || !info) return FA_STATUS_INVALID_ARGUMENT;
        lseend::SessionInfo s;
        const int st = h->set.state(session, &s, audio, mel, cmn_mean);
        if (st != FA_OK) return st;
        *info = fa_lseend_stream_session_info{s.audio_samples, s.mel_rows, s.cmn_count, s.decoder_mask_end,
                                              s.has_snapshot};
        return FA_STATUS_OK;
    });
}
