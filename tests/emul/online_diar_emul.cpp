// Host run of streaming speaker tracking's arithmetic (fluidaudio_b200/csrc/online_diar/online_diar_core.cuh; CPU
// test-suite only): one chunk of a session, from the logits and the model embeddings to the assigned ids, the segments
// and the database, with the functions the kernels call.
//   od_emul_new() / od_emul_free(p)
//   od_emul_chunk(p, logits, F, chunk_size, emb, offset, r, masks, need, assigned, seg_ids, seg_values)  segment count
//   od_emul_count(p, count, next_id), od_emul_read(p, speakers, current, raws)
#include "../../fluidaudio_b200/csrc/online_diar/online_diar_core.cuh"

#include <cstdint>
#include <cstring>
#include <vector>

using namespace fa::od;

namespace {

struct Emul {
    std::vector<Speaker> db;
    SessionMeta meta{0, 1};
    long long seq = 0;
};

struct CSpeaker {   // fa_od_speaker's layout
    int64_t key, numeric, update_count;
    float duration;
    int32_t named, has_numeric, permanent, raw_count;
};

} // namespace

extern "C" {

void *od_emul_new() { return new Emul(); }
void od_emul_free(void *p) { delete static_cast<Emul *>(p); }

int32_t od_emul_chunk(void *p, const float *logits, int32_t F, int64_t chunk_size, const float *emb, double offset,
                      const float *rr, float *masks, int32_t *need, int64_t *assigned, int64_t *seg_ids,
                      float *seg_values) {
    Emul &E = *static_cast<Emul *>(p);
    const Resolved r{rr[0], rr[1], rr[2], rr[3]};
    std::vector<unsigned char> bits((size_t)F);
    int clean[kLocal] = {0, 0, 0}, act[kLocal] = {0, 0, 0};
    for (int f = 0; f < F; ++f) {
        bits[f] = (unsigned char)class_bits(powerset_argmax(logits + (size_t)f * kClasses));
        for (int s = 0; s < kLocal; ++s) {
            clean[s] += clean_mask(bits[f], s);
            act[s] += (bits[f] >> s) & 1;
        }
    }
    const long long nm = masks_in_chunk(F, chunk_size);
    int nb = 0;
    for (int s = 0; s < kLocal; ++s) {
        for (int f = 0; f < F; ++f) masks[(size_t)s * F + f] = nm > 0 ? (float)clean_mask(bits[f % nm], s) : 0.0f;
        need[s] = !((float)clean[s] < r.min_active);
        nb |= need[s] << s;
    }
    float activity[kLocal];
    for (int s = 0; s < kLocal; ++s) activity[s] = (float)act[s];
    E.db.resize((size_t)E.meta.count + kLocal);
    long long idx[kLocal];
    assign_chunk(E.db.data(), E.meta, emb, activity, nb, r, E.seq, idx);
    E.seq += kLocal;
    E.db.resize((size_t)E.meta.count);
    float quality[kLocal];
    int has_id[kLocal];
    for (int s = 0; s < kLocal; ++s) {
        quality[s] = embedding_quality(emb + s * kDim);
        has_id[s] = idx[s] >= 0;
        assigned[2 * s] = idx[s] < 0 ? -1 : E.db[idx[s]].m.named;
        assigned[2 * s + 1] = idx[s] < 0 ? 0 : E.db[idx[s]].m.key;
    }
    std::vector<Segment> made((size_t)segment_bound(F)), out((size_t)segment_bound(F));
    const int n = chunk_segments(bits.data(), F, activity, has_id, quality, offset, r, made.data(), out.data());
    for (int k = 0; k < n; ++k) {
        const Speaker &S = E.db[idx[out[k].speaker]];
        seg_ids[2 * k] = S.m.named;
        seg_ids[2 * k + 1] = S.m.key;
        seg_values[3 * k] = out[k].start;
        seg_values[3 * k + 1] = out[k].end;
        seg_values[3 * k + 2] = out[k].quality;
    }
    return n;
}

void od_emul_count(void *p, int64_t *count, int64_t *next_id) {
    const Emul &E = *static_cast<Emul *>(p);
    *count = E.meta.count;
    *next_id = E.meta.next_id;
}

void od_emul_read(void *p, CSpeaker *out, float *cur, float *raws) {
    const Emul &E = *static_cast<Emul *>(p);
    for (size_t i = 0; i < E.db.size(); ++i) {
        const SpeakerMeta &m = E.db[i].m;
        out[i] = CSpeaker{m.key, m.numeric, m.update_count, m.duration, m.named, m.has_numeric, m.permanent,
                          m.raw_count};
        std::memcpy(cur + i * kDim, E.db[i].current, kDim * sizeof(float));
        for (int j = 0; j < kFifo; ++j)
            for (int k = 0; k < kDim; ++k) raws[(i * kFifo + j) * kDim + k] = j < m.raw_count ? raw_row(E.db[i], j)[k] : 0.0f;
    }
}

} // extern "C"
