// C ABI of streaming speaker tracking (declared in include/fluidaudio_b200_online_diar.h) over online_diar_kernels.cu.
// Every argument is checked here or in the session set before any copy or launch; every entry point that returns a
// status returns through guard() (c_abi.h), and the model-input calls lease the pooled call context
// (call_context.h).  The database operations run on a host copy of one session with online_diar_core.cuh's
// arithmetic and land whole, so a refused operation changes nothing.
#include "../../../include/fluidaudio_b200_online_diar.h"
#include "../c_abi.h"
#include "online_diar.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <memory>
#include <vector>

struct fa_od_databases {
    fa::od::Databases set;
};
static_assert(sizeof(fa::od::SpeakerView) == sizeof(fa_od_speaker), "fa_od_speaker's layout");

using namespace fa;
using namespace fa::od;

namespace {

// 16000 * Int(x.rounded()), where it stays below 2^40 samples
bool samples_of(float x, long long *out) {
    const double r = std::round((double)x);
    if (!(std::fabs(r) <= 68719476.0)) return false;   // NaN, inf, or 16000 * r beyond 2^40
    *out = 16000LL * (long long)r;
    return true;
}

int resolve(const fa_od_config *c, Resolved &r, fa_od_resolved *out, const char *where) {
    if (!c) return refuse("%s: cfg is NULL", where);
    long long chunk = 0, overlap = 0;
    if (!samples_of(c->chunk_duration, &chunk) || !samples_of(c->chunk_overlap, &overlap))
        return refuse("%s: chunk_duration %g or chunk_overlap %g is not finite or beyond 2^40 samples", where,
                      (double)c->chunk_duration, (double)c->chunk_overlap);
    if (chunk <= 0) return refuse("%s: chunk size %lld must be positive", where, chunk);
    if (chunk == overlap) return refuse("%s: the chunk step is 0", where);
    r = Resolved{f_mul(c->clustering_threshold, 1.2f), f_mul(c->clustering_threshold, 0.8f), c->min_speech_duration,
                 c->min_active_frames_count};
    if (out)
        *out = fa_od_resolved{r.speaker_threshold, r.embedding_threshold, r.min_speech, r.min_active, chunk,
                              chunk - overlap};
    return FA_OK;
}

bool offsets_ok(const int64_t *off, long long count) {
    if (!off || off[0] != 0) return false;
    for (long long i = 0; i < count; ++i)
        if (off[i + 1] < off[i] || off[i + 1] > (1LL << 62)) return false;
    return true;
}

int inputs(bool enroll, bool on_device, const float *audio, const int64_t *offsets, int32_t count,
           long long chunk_size, int frames, float *segmentation, float *waveform, float *mask) {
    const char *where = enroll ? "fa_od_enrollment_inputs" : "fa_od_chunk_inputs";
    if (count < 0 || !offsets_ok(offsets, count))
        return refuse("%s: count %d must be >= 0 with count + 1 offsets from 0, non-decreasing", where, count);
    if (!enroll && !(chunk_size > 0 && chunk_size <= (1LL << 40)))
        return refuse("%s: chunk_size %lld is outside 1 .. 2^40", where, chunk_size);
    if (enroll && !(frames >= 1 && frames <= (1 << 20))) return refuse("%s: frames %d is outside 1 .. 2^20", where, frames);
    if (count > 0 && (!waveform || (enroll ? !mask : !segmentation)))
        return refuse("%s: an output is NULL", where);
    if (offsets[count] > 0 && !audio) return refuse("%s: audio is NULL with %lld samples", where, (long long)offsets[count]);
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) {
        return inputs_call(C, on_device, audio, offsets, count, enroll ? 0 : chunk_size, segmentation, waveform, mask,
                           enroll ? frames : 0);
    });
}

int embedding_inputs(fa_od_databases *h, int32_t count, const int32_t *sessions, const float *logits,
                     const fa_od_config *cfg, bool device, float *masks, int32_t *need) {
    if (!h) return refuse("fa_od_embedding_inputs: h is NULL");
    Resolved r{};
    fa_od_resolved o{};
    const int st = resolve(cfg, r, &o, "fa_od_embedding_inputs");
    if (st != FA_OK) return st;
    return h->set.embedding_inputs(count, sessions, logits, o.chunk_size, r, device, masks, need);
}

int advance(fa_od_databases *h, int32_t count, const int32_t *sessions, const float *emb, const double *offsets,
            const fa_od_config *cfg, bool device, int64_t *assigned, int32_t *seg_counts, int64_t *seg_ids,
            float *seg_values) {
    if (!h) return refuse("fa_od_advance: h is NULL");
    Resolved r{};
    const int st = resolve(cfg, r, nullptr, "fa_od_advance");
    if (st != FA_OK) return st;
    return h->set.advance(count, sessions, emb, offsets, r, device, assigned, seg_counts, seg_ids, seg_values);
}

// ---- database operations on a host copy of one session
long long find(const std::vector<Speaker> &db, int named, long long key) {
    for (size_t i = 0; i < db.size(); ++i)
        if (db[i].m.named == named && db[i].m.key == key) return (long long)i;
    return -1;
}

// nextSpeakerId after reset(keepIfPermanent: true): one past the largest numeric id left, at least 1
long long next_after(const std::vector<Speaker> &db) {
    long long most = 0;
    for (const Speaker &s : db)
        if (s.m.has_numeric) most = std::max(most, s.m.numeric);
    return most + 1;
}

// Speaker.mergeWith(other): the raws of both, the 50 most recent when more (newest first), then the mean
void merge_into(Speaker &d, const Speaker &o) {
    std::vector<std::pair<long long, const float *>> all;
    for (int j = 0; j < d.m.raw_count; ++j) all.emplace_back(d.m.raw_seq[(d.m.raw_head + j) % kFifo], raw_row(d, j));
    for (int j = 0; j < o.m.raw_count; ++j) all.emplace_back(o.m.raw_seq[(o.m.raw_head + j) % kFifo], raw_row(o, j));
    if (all.size() > (size_t)kFifo) {
        std::stable_sort(all.begin(), all.end(), [](const auto &a, const auto &b) { return a.first > b.first; });
        all.resize(kFifo);
    }
    Speaker n = d;
    for (size_t j = 0; j < all.size(); ++j) {
        std::copy(all[j].second, all[j].second + kDim, n.raw[j]);
        n.m.raw_seq[j] = all[j].first;
    }
    n.m.raw_head = 0;
    n.m.raw_count = (int)all.size();
    n.m.duration = f_add(d.m.duration, o.m.duration);
    recalculate(n);
    n.m.update_count = d.m.update_count + o.m.update_count;
    d = n;
}

void reset(std::vector<Speaker> &db, SessionMeta &meta, bool keep) {
    if (!keep) {
        db.clear();
        meta = SessionMeta{0, 1};
        return;
    }
    db.erase(std::remove_if(db.begin(), db.end(), [](const Speaker &s) { return !s.m.permanent; }), db.end());
    meta = SessionMeta{(long long)db.size(), next_after(db)};
}

template <typename Op> int with_db(fa_od_databases *h, int32_t session, const char *where, Op &&op) {
    if (!h) return refuse("%s: h is NULL", where);
    Databases &D = h->set;
    long long count = 0, next_id = 0;
    int st = D.speaker_count(session, &count, &next_id);
    if (st != FA_OK) return st;
    std::vector<Speaker> db;
    st = D.load(session, db);
    if (st != FA_OK) return st;
    SessionMeta meta{count, next_id};
    bool changed = false;
    st = op(db, meta, changed);
    if (st != FA_OK || !changed) return st;
    meta.count = (long long)db.size();
    return D.write(session, db, meta);
}

int initialize(fa_od_databases *h, int32_t session, int32_t count, const fa_od_speaker *sp, const float *current,
               const float *raws, int32_t mode, int32_t preserve) {
    const char *where = "fa_od_initialize";
    if (count < 0 || (count > 0 && (!sp || !current))) return refuse("%s: count %d with speakers or current NULL", where, count);
    if (mode < FA_OD_MODE_RESET || mode > FA_OD_MODE_SKIP) return refuse("%s: mode %d is unknown", where, mode);
    long long rows = 0;
    for (int i = 0; i < count; ++i) {
        if (sp[i].raw_count < 0 || sp[i].raw_count > kFifo || (sp[i].named != 0 && sp[i].named != 1))
            return refuse("%s: speaker %d has raw_count %d or named %d out of range", where, i, sp[i].raw_count, sp[i].named);
        if (!sp[i].named && !(sp[i].has_numeric && sp[i].numeric == sp[i].key))
            return refuse("%s: speaker %d has a canonical id whose numeric value is not its key", where, i);
        for (int j = 0; j < i; ++j)
            if (sp[j].named == sp[i].named && sp[j].key == sp[i].key)
                return refuse("%s: speakers %d and %d have the same id", where, j, i);
        rows += sp[i].raw_count;
    }
    if (rows > 0 && !raws) return refuse("%s: raws is NULL with %lld rows", where, rows);
    return with_db(h, session, where, [&](std::vector<Speaker> &db, SessionMeta &meta, bool &changed) {
        changed = true;
        if (mode == FA_OD_MODE_RESET) reset(db, meta, preserve != 0);
        const long long seq0 = h->set.next_seq(rows);
        long long most = 0, row = 0;
        for (int i = 0; i < count; ++i) {
            Speaker s{};   // Speaker.init, then its raws through RawEmbedding.init
            l2_normalize(current + (size_t)i * kDim, s.current);
            s.m.key = sp[i].key;
            s.m.named = sp[i].named;
            s.m.numeric = sp[i].numeric;
            s.m.has_numeric = sp[i].has_numeric != 0;
            s.m.duration = sp[i].duration;
            s.m.update_count = sp[i].update_count;
            s.m.permanent = sp[i].permanent != 0;
            const int nr = sp[i].raw_count;
            for (int j = 0; j < nr; ++j) {
                const int at = s.m.raw_count++;
                l2_normalize(raws + (size_t)(row + j) * kDim, s.raw[at]);
                s.m.raw_seq[at] = seq0 + row + j;
            }
            row += nr;
            const long long at = find(db, s.m.named, s.m.key);
            if (at >= 0) {
                const bool locked = db[at].m.permanent && preserve;
                if (mode == FA_OD_MODE_SKIP || locked) continue;
                if (mode == FA_OD_MODE_MERGE) merge_into(db[at], s);
                else db[at] = s;
            } else {
                db.push_back(s);
            }
            if (s.m.has_numeric) most = std::max(most, s.m.numeric);
        }
        meta.next_id = most + 1;
        return FA_OK;
    });
}

// upsertSpeaker: an existing id takes the fields as given (its current embedding unnormalised, permanence only ever
// set); a new one is Speaker.init of them, appended, and moves nextSpeakerId past a numeric id
int upsert(fa_od_databases *h, int32_t session, const fa_od_speaker *sp, const float *current, const float *raws) {
    const char *where = "fa_od_upsert";
    if (!sp || !current) return refuse("%s: speaker or current is NULL", where);
    if (sp->raw_count < 0 || sp->raw_count > kFifo || (sp->named != 0 && sp->named != 1))
        return refuse("%s: raw_count %d or named %d out of range", where, sp->raw_count, sp->named);
    if (!sp->named && !(sp->has_numeric && sp->numeric == sp->key))
        return refuse("%s: a canonical id whose numeric value is not its key", where);
    if (sp->raw_count > 0 && !raws) return refuse("%s: raws is NULL with %d rows", where, sp->raw_count);
    return with_db(h, session, where, [&](std::vector<Speaker> &db, SessionMeta &meta, bool &changed) {
        changed = true;
        const long long seq0 = h->set.next_seq(sp->raw_count);
        const long long at = find(db, sp->named, sp->key);
        Speaker s = at >= 0 ? db[at] : Speaker{};
        if (at >= 0) {
            std::copy(current, current + kDim, s.current);
            s.m.permanent = s.m.permanent || sp->permanent;
        } else {
            l2_normalize(current, s.current);
            s.m.key = sp->key;
            s.m.named = sp->named;
            s.m.numeric = sp->numeric;
            s.m.has_numeric = sp->has_numeric != 0;
            s.m.permanent = sp->permanent != 0;
        }
        s.m.duration = sp->duration;
        s.m.update_count = sp->update_count;
        s.m.raw_head = 0;
        s.m.raw_count = sp->raw_count;
        for (int j = 0; j < sp->raw_count; ++j) {
            l2_normalize(raws + (size_t)j * kDim, s.raw[j]);
            s.m.raw_seq[j] = seq0 + j;
        }
        if (at >= 0) {
            db[at] = s;
        } else {
            db.push_back(s);
            if (s.m.has_numeric) meta.next_id = std::max(meta.next_id, s.m.numeric + 1);
        }
        return FA_OK;
    });
}

} // namespace

FA_API fa_status fa_od_upsert(fa_od_databases *h, int32_t session, const fa_od_speaker *speaker, const float *current,
                              const float *raws) {
    return guard(__func__, [&] { return upsert(h, session, speaker, current, raws); });
}

FA_API void fa_od_default_config(fa_od_config *cfg) {
    if (cfg) *cfg = fa_od_config{0.7f, 1.0f, 2.0f, 0.5f, -1, 10.0f, 10.0f, 0.0f};
}

FA_API fa_status fa_od_resolve(const fa_od_config *cfg, fa_od_resolved *out) {
    return guard(__func__, [&]() -> int {
        if (!out) return refuse("fa_od_resolve: out is NULL");
        Resolved r{};
        return resolve(cfg, r, out, "fa_od_resolve");
    });
}

FA_API fa_status fa_od_chunk_inputs(const float *audio, const int64_t *offsets, int32_t count, int64_t chunk_size,
                                    float *segmentation, float *waveform) {
    return guard(__func__, [&] {
        return inputs(false, false, audio, offsets, count, chunk_size, 0, segmentation, waveform, nullptr);
    });
}

FA_API fa_status fa_od_chunk_inputs_device(const float *d_audio, const int64_t *offsets, int32_t count,
                                           int64_t chunk_size, float *d_segmentation, float *d_waveform) {
    return guard(__func__, [&] {
        return inputs(false, true, d_audio, offsets, count, chunk_size, 0, d_segmentation, d_waveform, nullptr);
    });
}

FA_API fa_status fa_od_enrollment_inputs(const float *audio, const int64_t *offsets, int32_t count, int32_t frames,
                                         float *waveform, float *mask) {
    return guard(__func__, [&] { return inputs(true, false, audio, offsets, count, 0, frames, nullptr, waveform, mask); });
}

FA_API fa_status fa_od_enrollment_inputs_device(const float *d_audio, const int64_t *offsets, int32_t count,
                                                int32_t frames, float *d_waveform, float *d_mask) {
    return guard(__func__, [&] {
        return inputs(true, true, d_audio, offsets, count, 0, frames, nullptr, d_waveform, d_mask);
    });
}

FA_API fa_status fa_od_create(int32_t frames, fa_od_databases **out) {
    return guard(__func__, [&]() -> int {
        if (!out) return refuse("fa_od_create: out is NULL");
        *out = nullptr;
        if (!(frames >= 1 && frames <= (1 << 20))) return refuse("fa_od_create: frames %d is outside 1 .. 2^20", frames);
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        std::unique_ptr<fa_od_databases> h(new fa_od_databases());
        const int st = h->set.init(frames);
        if (st != FA_OK) return st;
        *out = h.release();
        return FA_STATUS_OK;
    });
}

FA_API void fa_od_destroy(fa_od_databases *h) { delete h; }

FA_API fa_status fa_od_open(fa_od_databases *h, int32_t *session) {
    return guard(__func__, [&]() -> int {
        if (!h || !session) return refuse("fa_od_open: h or session is NULL");
        int id = -1;
        const int st = h->set.open(&id);
        if (st == FA_OK) *session = id;
        return st;
    });
}

FA_API fa_status fa_od_close(fa_od_databases *h, int32_t session) {
    return guard(__func__, [&]() -> int { return h ? h->set.close(session) : refuse("fa_od_close: h is NULL"); });
}

FA_API fa_status fa_od_embedding_inputs(fa_od_databases *h, int32_t count, const int32_t *sessions,
                                        const float *logits, const fa_od_config *cfg, float *masks, int32_t *need) {
    return guard(__func__, [&] { return embedding_inputs(h, count, sessions, logits, cfg, false, masks, need); });
}

FA_API fa_status fa_od_embedding_inputs_device(fa_od_databases *h, int32_t count, const int32_t *sessions,
                                               const float *d_logits, const fa_od_config *cfg, float *d_masks,
                                               int32_t *d_need) {
    return guard(__func__, [&] { return embedding_inputs(h, count, sessions, d_logits, cfg, true, d_masks, d_need); });
}

FA_API fa_status fa_od_advance(fa_od_databases *h, int32_t count, const int32_t *sessions, const float *embeddings,
                               const double *chunk_offsets, const fa_od_config *cfg, int64_t *assigned,
                               int32_t *seg_counts, int64_t *seg_ids, float *seg_values) {
    return guard(__func__, [&] {
        return advance(h, count, sessions, embeddings, chunk_offsets, cfg, false, assigned, seg_counts, seg_ids,
                       seg_values);
    });
}

FA_API fa_status fa_od_advance_device(fa_od_databases *h, int32_t count, const int32_t *sessions,
                                      const float *d_embeddings, const double *chunk_offsets, const fa_od_config *cfg,
                                      int64_t *d_assigned, int32_t *d_seg_counts, int64_t *d_seg_ids,
                                      float *d_seg_values) {
    return guard(__func__, [&] {
        return advance(h, count, sessions, d_embeddings, chunk_offsets, cfg, true, d_assigned, d_seg_counts, d_seg_ids,
                       d_seg_values);
    });
}

FA_API fa_status fa_od_query(fa_od_databases *h, int32_t session, int32_t count, const float *embeddings,
                             float *distances) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.query(session, count, embeddings, false, distances) : refuse("fa_od_query: h is NULL");
    });
}

FA_API fa_status fa_od_query_device(fa_od_databases *h, int32_t session, int32_t count, const float *d_embeddings,
                                    float *d_distances) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.query(session, count, d_embeddings, true, d_distances)
                 : refuse("fa_od_query_device: h is NULL");
    });
}

FA_API fa_status fa_od_speaker_count(fa_od_databases *h, int32_t session, int64_t *count, int64_t *next_id) {
    return guard(__func__, [&]() -> int {
        if (!h || !count || !next_id) return refuse("fa_od_speaker_count: h, count or next_id is NULL");
        long long c = 0, n = 0;
        const int st = h->set.speaker_count(session, &c, &n);
        if (st == FA_OK) {
            *count = c;
            *next_id = n;
        }
        return st;
    });
}

FA_API fa_status fa_od_read(fa_od_databases *h, int32_t session, fa_od_speaker *speakers, float *current,
                            float *raws) {
    return guard(__func__, [&]() -> int {
        return h ? h->set.read(session, reinterpret_cast<SpeakerView *>(speakers), current, raws)
                 : refuse("fa_od_read: h is NULL");
    });
}

FA_API fa_status fa_od_initialize(fa_od_databases *h, int32_t session, int32_t count, const fa_od_speaker *speakers,
                                  const float *current, const float *raws, int32_t mode,
                                  int32_t preserve_if_permanent) {
    return guard(__func__, [&] {
        return initialize(h, session, count, speakers, current, raws, mode, preserve_if_permanent);
    });
}

FA_API fa_status fa_od_remove(fa_od_databases *h, int32_t session, int32_t named, int64_t key,
                              int32_t keep_if_permanent, int32_t *removed) {
    return guard(__func__, [&]() -> int {
        if (!removed) return refuse("fa_od_remove: removed is NULL");
        *removed = 0;
        return with_db(h, session, "fa_od_remove", [&](std::vector<Speaker> &db, SessionMeta &, bool &changed) {
            const long long at = find(db, named, key);
            if (at < 0 || (keep_if_permanent && db[at].m.permanent)) return FA_OK;
            db.erase(db.begin() + at);
            changed = true;
            *removed = 1;
            return FA_OK;
        });
    });
}

FA_API fa_status fa_od_merge(fa_od_databases *h, int32_t session, int32_t source_named, int64_t source_key,
                             int32_t destination_named, int64_t destination_key, int32_t stop_if_permanent,
                             int32_t *merged) {
    return guard(__func__, [&]() -> int {
        if (!merged) return refuse("fa_od_merge: merged is NULL");
        *merged = 0;
        return with_db(h, session, "fa_od_merge", [&](std::vector<Speaker> &db, SessionMeta &, bool &changed) {
            const long long s = find(db, source_named, source_key), d = find(db, destination_named, destination_key);
            if (s < 0 || d < 0 || s == d || (stop_if_permanent && db[s].m.permanent)) return FA_OK;
            merge_into(db[d], db[s]);
            db.erase(db.begin() + s);
            changed = true;
            *merged = 1;
            return FA_OK;
        });
    });
}

FA_API fa_status fa_od_set_permanent(fa_od_databases *h, int32_t session, int32_t named, int64_t key,
                                     int32_t permanent, int32_t *found) {
    return guard(__func__, [&]() -> int {
        if (!found) return refuse("fa_od_set_permanent: found is NULL");
        *found = 0;
        return with_db(h, session, "fa_od_set_permanent", [&](std::vector<Speaker> &db, SessionMeta &, bool &changed) {
            const long long at = find(db, named, key);
            if (at < 0) return FA_OK;
            db[at].m.permanent = permanent != 0;
            changed = true;
            *found = 1;
            return FA_OK;
        });
    });
}

FA_API fa_status fa_od_reset(fa_od_databases *h, int32_t session, int32_t keep_if_permanent) {
    return guard(__func__, [&] {
        return with_db(h, session, "fa_od_reset", [&](std::vector<Speaker> &db, SessionMeta &meta, bool &changed) {
            reset(db, meta, keep_if_permanent != 0);
            changed = true;
            return FA_OK;
        });
    });
}
