// Sortformer streaming sessions (fa_sortformer_*): SortformerStreamingState (SortformerTypes.swift:270-327) for any
// number of sessions in HBM, advanced by SortformerStateUpdater.streamingUpdate (SortformerStateUpdater.swift:31-165).
//
// Every length of the state follows from coreFrames and the configuration, never from values, so the host mirrors the
// cache and FIFO lengths, whether spkcachePreds exists, the chunk count, the FIFO ring's head and which of the two cache
// buffers is current.  A push therefore checks and plans every session before anything runs, uploads one descriptor
// per session and issues one kernel launch (sortformer_kernels.cu); the host variant stages its arrays in the set's one
// staging buffer (HostStaging, fa_common.cuh), which adds their copies and one synchronisation.  Only the silence mean
// and count depend on values, and they stay on the device.
#include "sortformer_plan.h"

#include <algorithm>
#include <cmath>

namespace fa {
namespace sortformer {

static long long round_up(long long v, long long m) { return (v + m - 1) / m * m; }

void Arena::init(const Config &c) {
    long long off = 0;
    auto take = [&](long long floats) {
        const long long o = off;
        off += round_up(floats, 4);
        return o;
    };
    fifo = take((long long)c.fifo_rows() * kDims);
    fifo_preds = take((long long)c.fifo_rows() * kSpeakers);
    for (int b = 0; b < 2; ++b) {
        cache[b] = take((long long)c.cache_rows() * kDims);
        cache_preds[b] = take((long long)c.cache_rows() * kSpeakers);
    }
    mean = take(kDims);
    stride = round_up(off, 64);
}

int resolve_config(const Config &in, int max_core, Config &out) {
    Config c = in;
    // SortformerConfig.init (SortformerTypes.swift:239-254)
    c.chunk_len = std::max(1, c.chunk_len);
    c.spkcache_len = std::max(c.spkcache_len, (1 + c.sil_per_spk) * kSpeakers);
    c.update_period = std::max(std::min(c.update_period, c.fifo_len + c.chunk_len), c.chunk_len);
    c.max_core = max_core <= 0 ? c.chunk_len : max_core;
    if (c.left_context < 0 || c.right_context < 0 || c.fifo_len < 0 || c.sil_per_spk < 0 || c.spkcache_len > (1 << 20) ||
        c.fifo_len > (1 << 20) || c.max_core > (1 << 20)) {
        fa::set_error("sortformer config: contexts, fifoLen and spkcacheSilFramesPerSpk must be >= 0, lengths <= 2^20");
        return FA_INVALID_ARGUMENT;
    }
    for (float v : {c.silence_threshold, c.pred_score_threshold, c.scores_boost_latest, c.strong_boost_rate,
                     c.weak_boost_rate, c.min_pos_scores_rate})
        if (!std::isfinite(v)) {
            fa::set_error("sortformer config: every threshold, boost and rate must be finite");
            return FA_INVALID_ARGUMENT;
        }
    // a real permuted index must stay below the placeholder maxIndex (SortformerStateUpdater.swift:543-547)
    if ((long long)(c.cache_rows() + c.sil_per_spk) * kSpeakers >= kMaxIndex) {
        fa::set_error("sortformer config: (spkcacheLen + fifoLen + max_core + sil) * 4 = %lld reaches maxIndex %d",
                      (long long)(c.cache_rows() + c.sil_per_spk) * kSpeakers, kMaxIndex);
        return FA_INVALID_ARGUMENT;
    }
    const int per_spk = c.spkcache_len / kSpeakers - c.sil_per_spk;   // (:229)
    c.strong_k = scaled_count(per_spk, c.strong_boost_rate);
    c.weak_k = scaled_count(per_spk, c.weak_boost_rate);
    c.min_pos = scaled_count(per_spk, c.min_pos_scores_rate);
    out = c;
    return FA_OK;
}

int plan_step(const Config &c, int spk, int fifo, int has_preds, int emb_length, long long pred_rows, int lc, int rc,
              Step &out) {
    if (lc < 0 || rc < 0 || emb_length < 0 || pred_rows < 0) {
        fa::set_error("sortformer update: negative context (%d, %d), embedding length %d or prediction rows %lld", lc, rc,
                      emb_length, pred_rows);
        return FA_INVALID_ARGUMENT;
    }
    const int core = emb_length - lc - rc;   // (:62)
    if (core < 0 || core > c.max_core) {
        fa::set_error("sortformer update: coreFrames = %d - %d - %d = %d outside [0, max_core = %d]", emb_length, lc, rc,
                      core, c.max_core);
        return FA_INVALID_ARGUMENT;
    }
    // insufficientPredsLength (:50-53, :84-92): the tentative rows end last
    const long long chunk_end = (long long)spk + fifo + lc + core;
    if (chunk_end + rc > pred_rows) {
        fa::set_error("sortformer update: insufficientPredsLength: %lld prediction rows needed, %lld given",
                      chunk_end + rc, pred_rows);
        return FA_INVALID_ARGUMENT;
    }
    out = Step{core, 0, 0, 0, spk, fifo + core, has_preds};
    const int ctx = core + fifo;   // (:108-121)
    if (ctx > c.fifo_len) {
        const int pop = std::min(std::max(c.update_period, ctx - c.fifo_len), ctx);
        out.pop = pop;
        out.fifo_after = ctx - pop;
        out.spkcache_after = spk + pop;
        if (out.spkcache_after > c.spkcache_len) {
            out.compress = 1;
            out.init_preds = has_preds ? 0 : 1;
            out.has_preds_after = 1;
            out.spkcache_after = c.spkcache_len;
        }
    }
    return FA_OK;
}

int SortformerSet::init(const Config &resolved) {
    cfg = resolved;
    arena.init(cfg);
    int st = stream.create();
    if (st == FA_OK) st = set_update_smem(cfg);
    return st;
}

int SortformerSet::open(int *session) {
    auto grow = [&](int grown) { return grow_slots(table.slots(), grown, stream, d_state, arena.stride, d_silence, 1); };
    // SortformerStreamingState.init (SortformerTypes.swift:301-315): empty cache and FIFO, no predictions, mean zero
    auto init = [&](int id) -> int {
        FA_CUDA_TRY(cudaMemsetAsync(d_state.data() + (size_t)id * arena.stride + arena.mean, 0, kDims * sizeof(float),
                                    stream));
        FA_CUDA_TRY(cudaMemsetAsync(d_silence.data() + id, 0, sizeof(long long), stream));
        return FA_OK;
    };
    return table.open(16, grow, init, session);
}

int SortformerSet::close(int session) { return table.close(session, "sortformer"); }

int SortformerSet::update(int count, const int *sessions, const float *embs, int emb_rows, const float *preds,
                          int pred_rows, const int *emb_lengths, const int *left, const int *right, bool on_device,
                          float *confirmed, long long confirmed_len, float *tentative, long long tentative_len,
                          int64_t *confirmed_rows, int64_t *tentative_rows) {
    if (count < 0 || emb_rows < 0 || pred_rows < 0 ||
        (count > 0 && (!sessions || !emb_lengths || !confirmed_rows || !tentative_rows))) {
        fa::set_error("sortformer update: count, emb_rows and pred_rows must be >= 0; sessions, emb_lengths and the row "
                      "counts non-null");
        return FA_INVALID_ARGUMENT;
    }
    if (count == 0) return FA_OK;
    int st = table.check(count, sessions, "sortformer update");
    if (st != FA_OK) return st;
    std::vector<Step> step(count);
    std::vector<SortformerSession> next(count);
    std::vector<int> lcs(count), rcs(count);
    long long conf = 0, tent = 0;
    for (int i = 0; i < count; ++i) {
        const SortformerSession &m = table[sessions[i]];
        // SortformerDiarizer.swift:553-554: the streaming rule when no context is given
        lcs[i] = left ? left[i] : (m.chunks > 0 ? cfg.left_context : 0);
        rcs[i] = right ? right[i] : cfg.right_context;
        if (emb_lengths[i] > emb_rows) {
            fa::set_error("sortformer update: emb_lengths[%d] = %d exceeds emb_rows %d", i, emb_lengths[i], emb_rows);
            return FA_INVALID_ARGUMENT;
        }
        st = plan_step(cfg, m.spk_len, m.fifo_len, m.has_preds, emb_lengths[i], pred_rows, lcs[i], rcs[i], step[i]);
        if (st != FA_OK) return st;
        const Step &S = step[i];
        next[i] = SortformerSession{S.spkcache_after, S.fifo_after, (m.fifo_head + S.pop) % cfg.fifo_rows(),
                                    m.parity ^ S.compress, S.has_preds_after, m.chunks + 1};
        conf += S.core;
        tent += rcs[i];
    }
    if ((conf > 0 && (!confirmed || confirmed_len < conf * kSpeakers)) ||
        (tent > 0 && (!tentative || tentative_len < tent * kSpeakers))) {
        fa::set_error("sortformer update: outputs need %lld confirmed and %lld tentative floats, buffers hold %lld and %lld",
                      conf * kSpeakers, tent * kSpeakers, confirmed ? confirmed_len : 0, tentative ? tentative_len : 0);
        return FA_INVALID_ARGUMENT;
    }
    const long long emb_floats = (long long)count * emb_rows * kDims, pred_floats = (long long)count * pred_rows * kSpeakers;
    if ((emb_floats > 0 && !embs) || (pred_floats > 0 && !preds)) {
        fa::set_error("sortformer update: chunk_embs / preds are null");
        return FA_INVALID_ARGUMENT;
    }

    // ---- buffers and descriptors
    HostStaging H(!on_device, stream);
    const float *e, *p;
    float *c_out, *t_out;
    const size_t desc_bytes = (size_t)count * sizeof(UpdateJob);
    st = update_desc.reserve(std::max<size_t>(desc_bytes, 4096));
    if (st == FA_OK)
        st = H.carve(staging, [&](HostStaging::Layout &l) {
            e = l.in(embs, (size_t)emb_floats);
            p = l.in(preds, (size_t)pred_floats);
            c_out = l.out(confirmed, (size_t)(conf * kSpeakers));
            t_out = l.out(tentative, (size_t)(tent * kSpeakers));
        });
    if (st != FA_OK) return st;
    UpdateJob *hj = static_cast<UpdateJob *>(update_desc.host.data());
    long long co = 0, to = 0;
    for (int i = 0; i < count; ++i) {
        const int id = sessions[i];
        const SortformerSession &m = table[id];
        const Step &S = step[i];
        hj[i] = UpdateJob{(long long)id * arena.stride, id, (long long)i * emb_rows * kDims,
                          (long long)i * pred_rows * kSpeakers, co * kSpeakers, to * kSpeakers, m.spk_len, m.fifo_len,
                          m.fifo_head, m.parity, lcs[i], rcs[i], S.core, S.pop, S.compress, S.init_preds};
        co += S.core;
        to += rcs[i];
    }

    // ---- device work, on the handle's stream
    st = update_desc.upload(desc_bytes, stream);
    if (st == FA_OK)
        st = launch_update(cfg, arena, static_cast<const UpdateJob *>(update_desc.device.data()), count, e, p,
                           d_state.data(), d_silence.data(), c_out, t_out, stream);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(H.finish());

    table.commit(count, sessions, next.data());
    for (int i = 0; i < count; ++i) {
        confirmed_rows[i] = step[i].core;
        tentative_rows[i] = rcs[i];
    }
    return FA_OK;
}

int SortformerSet::model_inputs(int count, const int *sessions, bool on_device, float *spkcache, float *fifo,
                                int *spkcache_lengths, int *fifo_lengths) {
    if (count < 0 || (count > 0 && (!sessions || !spkcache || (!fifo && cfg.fifo_len > 0)))) {
        fa::set_error("sortformer model inputs: count must be >= 0, sessions / spkcache / fifo non-null");
        return FA_INVALID_ARGUMENT;
    }
    if (count == 0) return FA_OK;
    int st = table.check(count, sessions, "sortformer model inputs");
    if (st != FA_OK) return st;
    const size_t desc_bytes = (size_t)count * sizeof(InputJob);
    const long long cache_floats = (long long)count * cfg.spkcache_len * kDims;
    const long long fifo_floats = (long long)count * cfg.fifo_len * kDims;
    HostStaging H(!on_device, stream);
    float *c_out, *f_out;
    st = input_desc.reserve(std::max<size_t>(desc_bytes, 4096));
    if (st == FA_OK)
        st = H.carve(staging, [&](HostStaging::Layout &l) {
            c_out = l.out(spkcache, (size_t)cache_floats);
            f_out = l.out(fifo, (size_t)fifo_floats);
        });
    if (st != FA_OK) return st;
    InputJob *hj = static_cast<InputJob *>(input_desc.host.data());
    for (int i = 0; i < count; ++i) {
        const SortformerSession &m = table[sessions[i]];
        hj[i] = InputJob{(long long)sessions[i] * arena.stride, m.spk_len, m.fifo_len, m.fifo_head, m.parity};
        if (spkcache_lengths) spkcache_lengths[i] = m.spk_len;
        if (fifo_lengths) fifo_lengths[i] = m.fifo_len;
    }
    st = input_desc.upload(desc_bytes, stream);
    if (st == FA_OK)
        st = launch_inputs(cfg, arena, static_cast<const InputJob *>(input_desc.device.data()), count, d_state.data(), c_out,
                           f_out, stream);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int SortformerSet::state(int session, SessionInfo *info, float *spkcache, float *spkcache_preds, float *fifo,
                         float *fifo_preds, float *mean) {
    if (!table.valid(session) || !info) {
        fa::set_error("sortformer state: session %d is not open (or info is null)", session);
        return FA_INVALID_ARGUMENT;
    }
    const SortformerSession &m = table[session];
    const int id = session, FR = cfg.fifo_rows(), head = m.fifo_head, n = m.fifo_len;
    const float *st = d_state.data() + (size_t)id * arena.stride;
    auto d2h = [&](float *dst, const float *src, size_t floats) {
        return floats ? cudaMemcpyAsync(dst, src, floats * sizeof(float), cudaMemcpyDeviceToHost, stream) : cudaSuccess;
    };
    // the FIFO ring's rows [head, head + n) in two runs
    const int first = std::min(n, FR - head);
    if (spkcache) FA_CUDA_TRY(d2h(spkcache, st + arena.cache[m.parity], (size_t)m.spk_len * kDims));
    if (spkcache_preds && m.has_preds)
        FA_CUDA_TRY(d2h(spkcache_preds, st + arena.cache_preds[m.parity], (size_t)m.spk_len * kSpeakers));
    if (fifo) {
        FA_CUDA_TRY(d2h(fifo, st + arena.fifo + (size_t)head * kDims, (size_t)first * kDims));
        FA_CUDA_TRY(d2h(fifo + (size_t)first * kDims, st + arena.fifo, (size_t)(n - first) * kDims));
    }
    if (fifo_preds) {
        FA_CUDA_TRY(d2h(fifo_preds, st + arena.fifo_preds + (size_t)head * kSpeakers, (size_t)first * kSpeakers));
        FA_CUDA_TRY(d2h(fifo_preds + (size_t)first * kSpeakers, st + arena.fifo_preds, (size_t)(n - first) * kSpeakers));
    }
    if (mean) FA_CUDA_TRY(d2h(mean, st + arena.mean, kDims));
    long long sil = 0;
    FA_CUDA_TRY(cudaMemcpyAsync(&sil, d_silence.data() + id, sizeof(long long), cudaMemcpyDeviceToHost, stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    *info = SessionInfo{m.spk_len, n, m.has_preds, m.chunks > 0 ? 1 : 0, m.chunks, sil};
    return FA_OK;
}

} // namespace sortformer
} // namespace fa
