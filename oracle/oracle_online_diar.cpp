// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
//
// Sequential CPU restatement of streaming speaker tracking, in the shape of the Swift source: DiarizerManager's
// processChunkWithSpeakerTracking and createTimedSegments, EmbeddingExtractor's input buffers, and SpeakerManager's
// database (a list in insertion order standing in for the Dictionary) with Speaker's raw-embedding FIFO, EMA and
// mergeWith.  The vDSP reductions (vDSP_dotpr, vDSP_svesq) take the library's documented order: 32 left folds over
// elements l, l + 32, ..., then an xor butterfly at distances 16, 8, 4, 2, 1.  Raw-embedding timestamps are a per-
// session counter.  Built with -O2 -ffp-contract=off on baseline x86-64, so each operation is one IEEE float op.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <deque>
#include <utility>
#include <vector>

namespace {

constexpr int D = 256;
using Vec = std::vector<float>;

float vdsp_dot(const float *a, const float *b) {
    float lane[32];
    for (int l = 0; l < 32; ++l) {
        float s = a[l] * b[l];
        for (int k = 1; k < 8; ++k) s = s + a[l + 32 * k] * b[l + 32 * k];
        lane[l] = s;
    }
    for (int o = 16; o >= 1; o /= 2) {
        float next[32];
        for (int l = 0; l < 32; ++l) next[l] = lane[l] + lane[l ^ o];
        std::memcpy(lane, next, sizeof(lane));
    }
    return lane[0];
}

float smax(float x, float y) { return y >= x ? y : x; }   // Swift.max
float smin(float x, float y) { return y < x ? y : x; }    // Swift.min

Vec l2n(const Vec &x) {   // VDSPOperations.l2Normalize
    const float norm = smax(std::sqrt(vdsp_dot(x.data(), x.data())), 1e-12f);
    const float scale = 1.0f / norm;
    Vec y(D);
    for (int i = 0; i < D; ++i) y[i] = x[i] * scale;
    return y;
}

float cosine(const Vec &a, const Vec &b) {   // SpeakerUtilities.cosineDistance
    const float dot = vdsp_dot(a.data(), b.data());
    const float sa = vdsp_dot(a.data(), a.data()), sb = vdsp_dot(b.data(), b.data());
    if (!(sa > 0 && sb > 0)) return INFINITY;
    float sim;
    if (std::fabs(sa - 1.0f) <= 1e-3f && std::fabs(sb - 1.0f) <= 1e-3f) {
        sim = dot;
    } else {
        const float ma = std::sqrt(sa), mb = std::sqrt(sb);
        if (!(ma > 0 && mb > 0)) return INFINITY;
        sim = dot / (ma * mb);
    }
    return 1 - smin(smax(sim, -1.0f), 1.0f);
}

struct Raw {
    long long timestamp;
    Vec e;
};

struct Spk {
    int named = 0, has_numeric = 0;
    long long key = 0, numeric = 0, update_count = 1;
    Vec cur;
    float duration = 0;
    std::deque<Raw> raws;
    bool permanent = false;

    void recalculate() {
        if (raws.empty()) return;
        Vec avg(D, 0.0f);
        for (const Raw &r : raws)
            for (int i = 0; i < D; ++i) avg[i] += r.e[i];
        const float n = (float)raws.size();
        for (int i = 0; i < D; ++i) avg[i] /= n;
        cur = l2n(avg);
    }
    void add_raw(const Raw &r) {
        if (!(vdsp_dot(r.e.data(), r.e.data()) > 0.01f)) return;
        if (raws.size() >= 50) raws.pop_front();
        raws.push_back(r);
        recalculate();
    }
    void update_main(float dur, const Vec &e, long long ts) {
        if (!(vdsp_dot(e.data(), e.data()) > 0.01f)) return;
        const Vec ne = l2n(e);
        add_raw(Raw{ts, l2n(ne)});
        for (int i = 0; i < D; ++i) cur[i] = 0.9f * cur[i] + (1 - 0.9f) * ne[i];
        cur = l2n(cur);
        duration += dur;
        update_count += 1;
    }
    void merge_with(const Spk &o) {
        std::vector<Raw> all(raws.begin(), raws.end());
        all.insert(all.end(), o.raws.begin(), o.raws.end());
        if (all.size() > 50) {
            std::stable_sort(all.begin(), all.end(), [](const Raw &a, const Raw &b) { return a.timestamp > b.timestamp; });
            all.resize(50);
        }
        raws.assign(all.begin(), all.end());
        duration += o.duration;
        recalculate();
        update_count += o.update_count;
    }
};

struct CSpeaker {   // fa_od_speaker's layout
    int64_t key, numeric, update_count;
    float duration;
    int32_t named, has_numeric, permanent, raw_count;
};

struct Db {
    std::vector<Spk> db;   // the Dictionary, in insertion order
    long long next_id = 1, clock = 0;

    long long find(int named, long long key) const {
        for (size_t i = 0; i < db.size(); ++i)
            if (db[i].named == named && db[i].key == key) return (long long)i;
        return -1;
    }
    void reset(bool keep) {
        if (!keep) {
            db.clear();
            next_id = 1;
            return;
        }
        std::vector<Spk> kept;
        for (const Spk &s : db)
            if (s.permanent) kept.push_back(s);
        db = kept;
        long long most = 0;
        for (const Spk &s : db)
            if (s.has_numeric) most = std::max(most, s.numeric);
        next_id = most + 1;
    }
    // SpeakerManager.assignSpeaker; returns the speaker's index or -1
    long long assign(const Vec &e, float dur, const float *r) {
        const Vec n = l2n(e);
        float best = INFINITY;
        long long at = -1;
        for (size_t i = 0; i < db.size(); ++i) {
            const float d = cosine(n, db[i].cur);
            if (d < best) {
                best = d;
                at = (long long)i;
            }
        }
        if (at >= 0 && best < r[0]) {
            Spk &s = db[at];
            if (best < r[1]) {
                if (vdsp_dot(n.data(), n.data()) > 0.01f) s.update_main(dur, n, clock++);
            } else {
                s.duration += dur;
            }
            return at;
        }
        if (!(dur >= r[2])) return -1;
        const Vec ne = l2n(n);
        Spk s;
        s.key = s.numeric = next_id++;
        s.has_numeric = 1;
        s.cur = l2n(ne);
        s.duration = dur;
        s.add_raw(Raw{clock++, l2n(ne)});
        const long long old = find(0, s.key);
        if (old >= 0) {
            db[old] = s;
            return old;
        }
        db.push_back(s);
        return (long long)db.size() - 1;
    }
};

} // namespace

extern "C" {

void *oracle_od_new() { return new Db(); }
void oracle_od_free(void *p) { delete static_cast<Db *>(p); }

// The segmentation input (chunk_size > 0) and the embedding waveform row 0 of one clip; for enrollment (chunk_size 0)
// the waveform and the all-ones mask of F entries
void oracle_od_inputs(const float *audio, int64_t n, int64_t chunk_size, int32_t F, float *seg, float *wave,
                      float *mask) {
    std::vector<float> padded;
    if (chunk_size > 0) {   // chunkBuffer: the chunk zero-padded to chunkSize
        padded.assign((size_t)std::min<int64_t>(chunk_size, 1 << 22), 0.0f);
        const int64_t copy = std::min(n, chunk_size);
        for (int64_t i = 0; i < copy && i < (int64_t)padded.size(); ++i) padded[i] = audio[i];
        for (int j = 0; j < 160000; ++j) seg[j] = j < (int64_t)padded.size() ? padded[j] : 0.0f;
    } else {
        padded.assign(audio, audio + std::min<int64_t>(n, 480000));
    }
    const int64_t count = chunk_size > 0 ? chunk_size : n;   // the audio's count as getEmbeddings sees it
    std::vector<float> buf(480000, 0.0f);                    // [3, 160000], zero-cleared
    const int64_t copy = std::min<int64_t>(count, 480000);
    for (int64_t i = 0; i < copy; ++i) buf[i] = i < (int64_t)padded.size() ? padded[i] : 0.0f;
    if (count > 0) {
        int64_t sc = count;
        while (sc < 160000) {
            const int64_t c = std::min(sc, 160000 - sc);
            for (int64_t i = 0; i < c; ++i) buf[sc + i] = buf[i];
            sc += c;
        }
    }
    std::memcpy(wave, buf.data(), 160000 * sizeof(float));
    if (mask) {
        const int64_t nm = std::min<int64_t>((F * count + 80000) / 160000, F);
        for (int f = 0; f < F; ++f) mask[f] = 0.0f;
        if (nm > 0) {
            for (int64_t f = 0; f < nm; ++f) mask[f] = 1.0f;
            int64_t c = nm;
            while (c < F) {
                const int64_t k = std::min(c, F - c);
                for (int64_t i = 0; i < k; ++i) mask[c + i] = mask[i];
                c += k;
            }
        }
    }
}

// One chunk of processChunkWithSpeakerTracking after the two models.  r: speakerThreshold, embeddingThreshold,
// minSpeechDuration, minActiveFramesCount.  Returns the segment count.
int32_t oracle_od_chunk(void *p, const float *logits, int32_t F, int64_t chunk_size, const float *model_emb,
                        double offset, const float *r, float *masks_out, int32_t *need_out, int64_t *assigned_out,
                        int64_t *seg_ids, float *seg_values) {
    Db &S = *static_cast<Db *>(p);
    static const int powerset[7][2] = {{-1, -1}, {0, -1}, {1, -1}, {2, -1}, {0, 1}, {0, 2}, {1, 2}};
    std::vector<std::vector<float>> bin((size_t)F, std::vector<float>(3, 0.0f));
    for (int f = 0; f < F; ++f) {
        const float *x = logits + (size_t)f * 7;
        float mv = x[0];
        int mi = 0;
        for (int c = 1; c < 7; ++c)
            if (x[c] > mv) {
                mv = x[c];
                mi = c;
            }
        for (int k = 0; k < 2; ++k)
            if (powerset[mi][k] >= 0) bin[f][powerset[mi][k]] = 1.0f;
    }
    // clean-frame masks and getEmbeddings
    std::vector<std::vector<float>> masks(3, std::vector<float>((size_t)F));
    for (int s = 0; s < 3; ++s)
        for (int f = 0; f < F; ++f) {
            const float sum = bin[f][0] + bin[f][1] + bin[f][2];
            masks[s][f] = bin[f][s] * (sum < 2.0f ? 1.0f : 0.0f);
        }
    const long long nm = std::min<long long>(((long long)F * chunk_size + 80000) / 160000, F);
    std::vector<Vec> emb(3, Vec(D, 0.0f));
    for (int s = 0; s < 3; ++s) {
        float act = 0;
        for (float v : masks[s]) act += v;
        need_out[s] = !(act < r[3]);
        for (int f = 0; f < F; ++f) masks_out[(size_t)s * F + f] = nm > 0 ? masks[s][f % nm] : 0.0f;
        if (need_out[s]) emb[s].assign(model_emb + s * D, model_emb + (s + 1) * D);
    }
    float activity[3] = {0, 0, 0};
    for (int s = 0; s < 3; ++s)
        for (int f = 0; f < F; ++f) activity[s] += bin[f][s];
    long long ids[3] = {-1, -1, -1};
    for (int s = 0; s < 3; ++s) {
        if (!(activity[s] > r[3])) continue;
        bool ok = true;   // AudioValidation.validateEmbedding
        float ss = 0;
        for (float v : emb[s]) {
            ok = ok && std::isfinite(v);
            ss = ss + v * v;
        }
        if (!ok || !(std::sqrt(ss) > 0.1f)) continue;
        ids[s] = S.assign(emb[s], activity[s] * (float)0.016875, r);
    }
    for (int s = 0; s < 3; ++s) {
        assigned_out[2 * s] = ids[s] < 0 ? -1 : S.db[ids[s]].named;
        assigned_out[2 * s + 1] = ids[s] < 0 ? 0 : S.db[ids[s]].key;
    }
    struct Seg {
        int s;
        float start, end, q;
    };
    std::vector<Seg> segs;
    for (int s = 0; s < 3; ++s) {
        if (activity[s] < r[3]) continue;
        const float quality = smin(1.0f, std::sqrt(vdsp_dot(emb[s].data(), emb[s].data())) / 10.0f);
        auto emit = [&](int a, int b) {
            if (ids[s] < 0) return;
            const double t0 = offset + (double)a * 0.016875, t1 = offset + (double)b * 0.016875;
            if ((float)(t1 - t0) < r[2]) return;
            segs.push_back(Seg{s, (float)t0, (float)t1, quality * (activity[s] / (float)(b - a))});
        };
        bool on = false;
        int start = 0;
        for (int f = 0; f < F; ++f) {
            float th = 0.3f;
            for (int o = 0; o < 3; ++o)
                if (o != s && bin[f][o] > 0.3f) {
                    th = 0.15f;
                    break;
                }
            if (bin[f][s] > th && !on) {
                on = true;
                start = f;
            } else if (bin[f][s] <= th && on) {
                emit(start, f);
                on = false;
            }
        }
        if (on) emit(start, F);
    }
    std::stable_sort(segs.begin(), segs.end(), [](const Seg &a, const Seg &b) { return a.start < b.start; });
    for (size_t k = 0; k < segs.size(); ++k) {
        const Spk &sp = S.db[ids[segs[k].s]];
        seg_ids[2 * k] = sp.named;
        seg_ids[2 * k + 1] = sp.key;
        seg_values[3 * k] = segs[k].start;
        seg_values[3 * k + 1] = segs[k].end;
        seg_values[3 * k + 2] = segs[k].q;
    }
    return (int32_t)segs.size();
}

void oracle_od_count(void *p, int64_t *count, int64_t *next_id) {
    const Db &S = *static_cast<Db *>(p);
    *count = (int64_t)S.db.size();
    *next_id = S.next_id;
}

void oracle_od_read(void *p, CSpeaker *out, float *cur, float *raws) {
    const Db &S = *static_cast<Db *>(p);
    for (size_t i = 0; i < S.db.size(); ++i) {
        const Spk &s = S.db[i];
        out[i] = CSpeaker{s.key, s.numeric, s.update_count, s.duration, s.named, s.has_numeric, s.permanent,
                          (int32_t)s.raws.size()};
        std::memcpy(cur + i * D, s.cur.data(), D * sizeof(float));
        for (int j = 0; j < 50; ++j)
            for (int k = 0; k < D; ++k) raws[(i * 50 + j) * D + k] = j < (int)s.raws.size() ? s.raws[j].e[k] : 0.0f;
    }
}

// initializeKnownSpeakers(_:mode:preserveIfPermanent:); mode 0 reset, 1 merge, 2 overwrite, 3 skip
void oracle_od_initialize(void *p, int32_t n, const CSpeaker *sp, const float *cur, const float *raws, int32_t mode,
                          int32_t preserve) {
    Db &S = *static_cast<Db *>(p);
    if (mode == 0) S.reset(preserve != 0);
    long long most = 0, row = 0;
    for (int i = 0; i < n; ++i) {
        Spk s;
        s.key = sp[i].key;
        s.named = sp[i].named;
        s.numeric = sp[i].numeric;
        s.has_numeric = sp[i].has_numeric;
        s.cur = l2n(Vec(cur + (size_t)i * D, cur + (size_t)(i + 1) * D));
        s.duration = sp[i].duration;
        s.update_count = sp[i].update_count;
        s.permanent = sp[i].permanent != 0;
        for (int j = 0; j < sp[i].raw_count; ++j, ++row)
            s.raws.push_back(Raw{S.clock++, l2n(Vec(raws + (size_t)row * D, raws + (size_t)(row + 1) * D))});
        const long long at = S.find(s.named, s.key);
        if (at >= 0) {
            if (mode == 3 || (S.db[at].permanent && preserve)) continue;
            if (mode == 1) S.db[at].merge_with(s);
            else S.db[at] = s;
        } else {
            S.db.push_back(s);
        }
        if (s.has_numeric) most = std::max(most, s.numeric);
    }
    S.next_id = most + 1;
}

// upsertSpeaker: an existing id takes the fields (currentEmbedding as given); a new one is Speaker.init of them
void oracle_od_upsert(void *p, const CSpeaker *sp, const float *cur, const float *raws) {
    Db &S = *static_cast<Db *>(p);
    std::deque<Raw> rs;
    for (int j = 0; j < sp->raw_count; ++j) rs.push_back(Raw{S.clock++, l2n(Vec(raws + (size_t)j * D, raws + (size_t)(j + 1) * D))});
    const long long at = S.find(sp->named, sp->key);
    if (at >= 0) {
        Spk &s = S.db[at];
        s.cur.assign(cur, cur + D);
        s.duration = sp->duration;
        s.raws = rs;
        s.update_count = sp->update_count;
        if (sp->permanent) s.permanent = true;
        return;
    }
    Spk s;
    s.key = sp->key;
    s.named = sp->named;
    s.numeric = sp->numeric;
    s.has_numeric = sp->has_numeric;
    s.cur = l2n(Vec(cur, cur + D));
    s.duration = sp->duration;
    s.permanent = sp->permanent != 0;
    s.raws = rs;
    s.update_count = sp->update_count;
    S.db.push_back(s);
    if (s.has_numeric) S.next_id = std::max(S.next_id, s.numeric + 1);
}

int32_t oracle_od_remove(void *p, int32_t named, int64_t key, int32_t keep) {
    Db &S = *static_cast<Db *>(p);
    const long long at = S.find(named, key);
    if (at < 0 || (keep && S.db[at].permanent)) return 0;
    S.db.erase(S.db.begin() + at);
    return 1;
}

int32_t oracle_od_merge(void *p, int32_t sn, int64_t sk, int32_t dn, int64_t dk, int32_t stop) {
    Db &S = *static_cast<Db *>(p);
    if (sn == dn && sk == dk) return 0;
    const long long s = S.find(sn, sk), d = S.find(dn, dk);
    if (s < 0 || d < 0 || (stop && S.db[s].permanent)) return 0;
    S.db[d].merge_with(S.db[s]);
    S.db.erase(S.db.begin() + s);
    return 1;
}

int32_t oracle_od_set_permanent(void *p, int32_t named, int64_t key, int32_t flag) {
    Db &S = *static_cast<Db *>(p);
    const long long at = S.find(named, key);
    if (at < 0) return 0;
    S.db[at].permanent = flag != 0;
    return 1;
}

void oracle_od_reset(void *p, int32_t keep) { static_cast<Db *>(p)->reset(keep != 0); }

void oracle_od_query(void *p, int32_t n, const float *emb, float *dist) {
    const Db &S = *static_cast<Db *>(p);
    for (int q = 0; q < n; ++q) {
        const Vec e(emb + (size_t)q * D, emb + (size_t)(q + 1) * D);
        for (size_t i = 0; i < S.db.size(); ++i) dist[(size_t)q * S.db.size() + i] = cosine(e, S.db[i].cur);
    }
}

} // extern "C"
