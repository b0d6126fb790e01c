// Streaming speaker tracking on the GPU (online_diar.h, online_diar_core.cuh).
//
// Each session owns one slot: a SessionMeta header, capacity_ Speaker records (the current embedding, the 50-deep
// FIFO of raw embeddings and the metadata, about 52 KB each) in insertion order, and the chunk staged between the two
// calls around the embedding model (its binarized frames and need bits).  Every session slot holds the same speaker
// capacity; before a call that can add speakers the host makes room for three more in every session it names, doubling
// the capacity, so a session grows without a cap other than memory.  One launch per call:
//   od_inputs_kernel            the segmentation model's 160 000 samples and the embedding model's repeat-padded
//                               waveform, per chunk or enrollment clip
//   od_embedding_inputs_kernel  one CTA per session: powerset decoding, the clean-frame masks repeat-padded to the
//                               embedding model's row, and the need flags
//   od_advance_kernel           one CTA per session: assignSpeaker for local speakers 0, 1, 2 in order (the distance
//                               scan split across the warps, the FIFO mean thread-per-dimension), then the segments
//   od_query_kernel             one CTA per query: the cosine distance to every speaker of a session
#include "online_diar.h"

#include <algorithm>
#include <cstring>
#include <cuda_runtime.h>

namespace fa {
namespace od {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// tree_dot (online_diar_core.cuh) on one warp: every lane returns the same sum
__device__ float warp_dot(const float *a, const float *b) {
    const int l = threadIdx.x & 31;
    float s = f_mul(a[l], b[l]);
    for (int k = 1; k < 8; ++k) s = f_add(s, f_mul(a[l + 32 * k], b[l + 32 * k]));
    for (int o = 16; o >= 1; o >>= 1) s = f_add(s, __shfl_xor_sync(0xffffffffu, s, o));
    return s;
}

// l2_normalize on one warp (x and y may be the same array)
__device__ void warp_normalize(const float *x, float *y) {
    const float scale = norm_scale(warp_dot(x, x));
    const int l = threadIdx.x & 31;
    float v[8];
    for (int k = 0; k < 8; ++k) v[k] = f_mul(x[l + 32 * k], scale);
    __syncwarp();
    for (int k = 0; k < 8; ++k) y[l + 32 * k] = v[k];
    __syncwarp();
}

struct InputJob {
    long long src, n, period;   // the clip's first sample, the samples taken and the waveform's repeat period
};

__global__ void __launch_bounds__(kThreads)
    od_inputs_kernel(const InputJob *__restrict__ jobs, const float *__restrict__ audio, float *__restrict__ seg,
                     float *__restrict__ wave, float *__restrict__ mask, int frames, int count) {
    for (int b = blockIdx.y; b < count; b += gridDim.y) {   // gridDim.y is at most 65 535: clips stride over it
        const InputJob J = jobs[b];
        const float *x = audio + J.src;
        const size_t row = (size_t)b * kModelSamples;
        for (int j = blockIdx.x * kThreads + threadIdx.x; j < kModelSamples; j += gridDim.x * kThreads) {
            if (seg) seg[row + j] = j < J.n ? x[j] : 0.0f;
            const long long k = J.period >= kModelSamples ? j : J.period > 0 ? j % J.period : -1;
            wave[row + j] = k >= 0 && k < J.n ? x[k] : 0.0f;
        }
        if (mask && blockIdx.x == 0) {   // extractSpeakerEmbedding's all-ones mask, repeat-padded
            const float v = masks_in_chunk(frames, J.n) > 0 ? 1.0f : 0.0f;
            for (int f = threadIdx.x; f < frames; f += kThreads) mask[(size_t)b * frames + f] = v;
        }
    }
}

__global__ void __launch_bounds__(kThreads)
    od_embedding_inputs_kernel(const int *__restrict__ slots, const float *__restrict__ logits, int frames,
                               long long n_masks, float min_active, unsigned char *bits, float *__restrict__ masks,
                               int *__restrict__ need) {
    __shared__ int clean[kLocal];
    const int b = blockIdx.x;
    unsigned char *B = bits + (size_t)slots[b] * (frames + 1);
    if (threadIdx.x < kLocal) clean[threadIdx.x] = 0;
    __syncthreads();
    int c[kLocal] = {0, 0, 0};
    for (int f = threadIdx.x; f < frames; f += kThreads) {
        const int v = class_bits(powerset_argmax(logits + ((size_t)b * frames + f) * kClasses));
        B[f] = (unsigned char)v;
        for (int s = 0; s < kLocal; ++s) c[s] += clean_mask(v, s);
    }
    for (int s = 0; s < kLocal; ++s) atomicAdd(&clean[s], c[s]);
    __syncthreads();
    for (int s = 0; s < kLocal; ++s)
        for (int f = threadIdx.x; f < frames; f += kThreads)
            masks[((size_t)b * kLocal + s) * frames + f] = n_masks > 0 ? (float)clean_mask(B[f % n_masks], s) : 0.0f;
    if (threadIdx.x == 0) {   // getEmbeddings skips a speaker whose mask sums below minActivityThreshold
        int nb = 0;
        for (int s = 0; s < kLocal; ++s) {
            const int on = !((float)clean[s] < min_active);
            need[b * kLocal + s] = on;
            nb |= on << s;
        }
        B[frames] = (unsigned char)nb;
    }
}

struct AdvanceArgs {
    const int *slots;
    const float *emb;        // [count x 3 x 256]
    const double *offsets;   // chunk offsets, seconds
    Speaker *db;
    SessionMeta *meta;
    const unsigned char *bits;
    Segment *made;           // [count x bound] scratch
    SessionMeta *out_meta;   // [count]: the pushed sessions' headers in call order
    long long *assigned;     // [count x 3 x 2]
    int *seg_counts;
    long long *seg_ids;      // [count x bound x 2]
    float *seg_values;       // [count x bound x 3]
    long long capacity, bound, seq0;
    int frames;
    Resolved r;
};

__global__ void __launch_bounds__(kThreads) od_advance_kernel(AdvanceArgs a) {
    __shared__ float e[kDim], q[kDim], ne[kDim], t[kDim];
    __shared__ float wd[kWarps];
    __shared__ long long wi[kWarps];
    __shared__ int act[kLocal], go, op, add_ok;
    __shared__ long long target, canon, assigned[kLocal];
    __shared__ float ssq, duration;
    __shared__ SessionMeta M;
    const int b = blockIdx.x, tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
    const int slot = a.slots[b];
    Speaker *db = a.db + (size_t)slot * a.capacity;
    const unsigned char *B = a.bits + (size_t)slot * (a.frames + 1);
    if (tid < kLocal) act[tid] = 0;
    if (tid == 0) M = a.meta[slot];
    __syncthreads();
    int c[kLocal] = {0, 0, 0};
    for (int f = tid; f < a.frames; f += kThreads)
        for (int s = 0; s < kLocal; ++s) c[s] += (B[f] >> s) & 1;
    for (int s = 0; s < kLocal; ++s) atomicAdd(&act[s], c[s]);
    const int need = B[a.frames];
    __syncthreads();
    for (int s = 0; s < kLocal; ++s) {
        const float activity = (float)act[s];
        const bool ran = (need >> s) & 1;   // the embedding model ran for s: only then is its row read
        if (ran) e[tid] = a.emb[((size_t)b * kLocal + s) * kDim + tid];
        if (tid == 0) {
            assigned[s] = -1;
            canon = -1;
        }
        __syncthreads();
        if (tid == 0) go = activity > a.r.min_active && ran && valid_embedding(e);
        __syncthreads();
        if (!go) continue;
        if (w == 0) {
            warp_normalize(e, q);
            const float ss = warp_dot(q, q);
            if (lane == 0) ssq = ss;
        }
        __syncthreads();
        // findClosestSpeaker: each warp scans its speakers in order, then the warps' bests meet (ties: lower index)
        float bd = INFINITY;
        long long bi = -1;
        for (long long i = w; i < M.count; i += kWarps) {
            const float d = cosine_from(warp_dot(q, db[i].current), ssq, warp_dot(db[i].current, db[i].current));
            if (d < bd) {
                bd = d;
                bi = i;
            }
        }
        if (lane == 0) {
            wd[w] = bd;
            wi[w] = bi;
        }
        for (long long i = tid; i < M.count; i += kThreads)   // a speaker already holding the next new id
            if (!db[i].m.named && db[i].m.key == M.next_id) atomicMin((unsigned long long *)&canon, (unsigned long long)i);
        __syncthreads();
        if (tid == 0) {
            float d = INFINITY;
            long long i = -1;
            for (int k = 0; k < kWarps; ++k)
                if (wi[k] >= 0 && (i < 0 || wd[k] < d || (wd[k] == d && wi[k] < i))) {
                    d = wd[k];
                    i = wi[k];
                }
            duration = f_mul(activity, (float)kFrameStep);
            op = 0;   // 0: nothing stored, 1: updateMainEmbedding, 2: duration only, 3: createNewSpeaker
            if (i >= 0 && d < a.r.speaker_threshold) {
                target = assigned[s] = i;
                op = d < a.r.embedding_threshold ? (ssq > 0.01f ? 1 : 0) : 2;
            } else if (duration >= a.r.min_speech) {
                target = assigned[s] = canon >= 0 ? canon : M.count++;
                op = 3;
            }
            if (op == 3) {
                Speaker &S = db[target];
                S.m = SpeakerMeta{};
                S.m.key = S.m.numeric = M.next_id++;
                S.m.has_numeric = 1;
                S.m.update_count = 1;
                S.m.duration = duration;
            } else if (op == 2) {
                db[target].m.duration = f_add(db[target].m.duration, duration);
            }
        }
        __syncthreads();
        if (op == 0 || op == 2) continue;
        Speaker &S = db[target];
        // ne: the embedding normalised once more (updateMainEmbedding, or Speaker.init); t: RawEmbedding.init's row
        if (w == 0) {
            warp_normalize(q, ne);
            warp_normalize(ne, t);
            if (op == 3) {
                for (int k = 0; k < 8; ++k) S.current[lane + 32 * k] = t[lane + 32 * k];
            }
            const float ss = warp_dot(t, t);
            if (lane == 0) {
                add_ok = ss > 0.01f;
                if (add_ok) {   // addRawEmbedding's FIFO
                    if (S.m.raw_count >= kFifo) {
                        S.m.raw_head = (S.m.raw_head + 1) % kFifo;
                        --S.m.raw_count;
                    }
                    const int at = (S.m.raw_head + S.m.raw_count) % kFifo;
                    S.m.raw_seq[at] = a.seq0 + (long long)b * kLocal + s;
                    ++S.m.raw_count;
                }
            }
            __syncwarp();
        }
        __syncthreads();
        if (add_ok) {
            const int n = S.m.raw_count;
            S.raw[(S.m.raw_head + n - 1) % kFifo][tid] = t[tid];
            __syncthreads();
            float acc = 0.0f;   // recalculateMainEmbedding, thread-per-dimension in FIFO order
            for (int j = 0; j < n; ++j) acc = f_add(acc, S.raw[(S.m.raw_head + j) % kFifo][tid]);
            e[tid] = f_div(acc, (float)n);
            __syncthreads();
            if (w == 0) warp_normalize(e, e);
            __syncthreads();
            S.current[tid] = e[tid];
        }
        __syncthreads();
        if (op == 1) {   // the EMA after the raw mean, then its normalisation
            e[tid] = ema(S.current[tid], ne[tid]);
            __syncthreads();
            if (w == 0) warp_normalize(e, e);
            __syncthreads();
            S.current[tid] = e[tid];
            if (tid == 0) {
                S.m.duration = f_add(S.m.duration, duration);
                ++S.m.update_count;
            }
        }
        __syncthreads();
    }
    __syncthreads();
    if (tid < kLocal) {
        long long *o = a.assigned + ((size_t)b * kLocal + tid) * 2;
        const long long i = assigned[tid];
        o[0] = i < 0 ? -1 : db[i].m.named;
        o[1] = i < 0 ? 0 : db[i].m.key;
    }
    if (w == 0) {   // the quality of the embeddings that got an id, for their segments (the raw model outputs)
        for (int s = 0; s < kLocal; ++s) {
            if (assigned[s] < 0) continue;
            const float *x = a.emb + ((size_t)b * kLocal + s) * kDim;
            const float qual = swift_min(1.0f, f_div(f_sqrt(warp_dot(x, x)), 10.0f));
            if (lane == 0) t[s] = qual;
        }
    }
    __syncthreads();
    if (tid == 0) {
        a.meta[slot] = M;
        a.out_meta[b] = M;
        float activity[kLocal];
        int has_id[kLocal];
        for (int s = 0; s < kLocal; ++s) {
            activity[s] = (float)act[s];
            has_id[s] = assigned[s] >= 0;
        }
        Segment *out = a.made + (size_t)b * 2 * a.bound;
        const int n = chunk_segments(B, a.frames, activity, has_id, t, a.offsets[b], a.r, out + a.bound, out);
        a.seg_counts[b] = n;
        for (int k = 0; k < n; ++k) {
            const Speaker &S = db[assigned[out[k].speaker]];
            long long *id = a.seg_ids + ((size_t)b * a.bound + k) * 2;
            float *v = a.seg_values + ((size_t)b * a.bound + k) * 3;
            id[0] = S.m.named;
            id[1] = S.m.key;
            v[0] = out[k].start;
            v[1] = out[k].end;
            v[2] = out[k].quality;
        }
    }
}

__global__ void __launch_bounds__(kThreads)
    od_query_kernel(const Speaker *__restrict__ db, long long count, const float *__restrict__ queries,
                    float *__restrict__ distances) {
    const int w = threadIdx.x >> 5;
    const float *x = queries + (size_t)blockIdx.x * kDim;
    const float ssa = warp_dot(x, x);
    for (long long i = w; i < count; i += kWarps) {
        const float d = cosine_from(warp_dot(x, db[i].current), ssa, warp_dot(db[i].current, db[i].current));
        if ((threadIdx.x & 31) == 0) distances[(size_t)blockIdx.x * count + i] = d;
    }
}

int check_sessions(const SessionTable<Mirror> &table, int count, const int *sessions, const char *where) {
    if (count < 0 || (count > 0 && !sessions)) {
        set_error("%s: count %d must be >= 0 and sessions non-null", where, count);
        return FA_INVALID_ARGUMENT;
    }
    return table.check(count, sessions, where);
}

} // namespace

// ------------------------------------------------------------------------------------------------ sessions
int Databases::init(int frames) {
    frames_ = frames;
    return stream.create();
}

// Moves every slot into buffers of `slots` slots x `capacity` speakers.  Everything is allocated before anything is
// copied: a failed allocation changes nothing.
int Databases::grow(int slots, int capacity) {
    DeviceBuffer<Speaker> ndb;
    DeviceBuffer<SessionMeta> nmeta;
    DeviceBuffer<unsigned char> nbits;
    int st = ndb.grow((size_t)slots * capacity * sizeof(Speaker));
    if (st == FA_OK) st = nmeta.grow((size_t)slots * sizeof(SessionMeta));
    if (st == FA_OK) st = nbits.grow((size_t)slots * (frames_ + 1));
    if (st != FA_OK) return st;
    const int old = table.slots();
    if (old) {
        if (capacity_)
            FA_CUDA_TRY(cudaMemcpy2DAsync(ndb.data(), (size_t)capacity * sizeof(Speaker), d_db.data(),
                                          (size_t)capacity_ * sizeof(Speaker), (size_t)capacity_ * sizeof(Speaker),
                                          (size_t)old, cudaMemcpyDeviceToDevice, stream));
        FA_CUDA_TRY(cudaMemcpyAsync(nmeta.data(), d_meta.data(), (size_t)old * sizeof(SessionMeta),
                                    cudaMemcpyDeviceToDevice, stream));
        FA_CUDA_TRY(cudaMemcpyAsync(nbits.data(), d_bits.data(), (size_t)old * (frames_ + 1), cudaMemcpyDeviceToDevice,
                                    stream));
        FA_CUDA_TRY(cudaStreamSynchronize(stream));
    }
    d_db = std::move(ndb);
    d_meta = std::move(nmeta);
    d_bits = std::move(nbits);
    capacity_ = capacity;
    return FA_OK;
}

int Databases::reserve(int need_speakers) {
    if (need_speakers <= capacity_) return FA_OK;
    if (need_speakers > (1 << 30)) {
        set_error("online diarization: %d speakers in one session is beyond the library's limit", need_speakers);
        return FA_INVALID_ARGUMENT;
    }
    return grow(std::max(table.slots(), 1), std::max({need_speakers, 2 * capacity_, 4}));
}

int Databases::open(int *session) {
    auto grow_slots = [&](int grown) { return grow(grown, std::max(capacity_, 4)); };
    auto init = [&](int id) -> int {   // SpeakerManager(): an empty database, nextSpeakerId 1
        const SessionMeta m{0, 1};
        FA_CUDA_TRY(cudaMemcpyAsync(d_meta.data() + id, &m, sizeof(m), cudaMemcpyHostToDevice, stream));
        FA_CUDA_TRY(cudaStreamSynchronize(stream));
        table[id].meta = m;
        return FA_OK;
    };
    return table.open(64, grow_slots, init, session);
}

int Databases::close(int session) { return table.close(session, "fa_od_close"); }

int Databases::embedding_inputs(int count, const int *sessions, const float *logits, long long chunk_size,
                                const Resolved &r, bool device, float *masks, int32_t *need) {
    const char *where = "fa_od_embedding_inputs";
    int st = check_sessions(table, count, sessions, where);
    if (st != FA_OK) return st;
    if (count > 0 && (!logits || !masks || !need)) {
        set_error("%s: logits, masks and need must be non-null", where);
        return FA_INVALID_ARGUMENT;
    }
    if (count == 0) return FA_OK;
    st = desc.reserve(std::max<size_t>((size_t)count * sizeof(int), 4096));
    if (st != FA_OK) return st;
    HostStaging H(!device, stream);
    const float *k_l;
    float *k_m;
    int *k_n;
    st = H.carve(d_io, [&](HostStaging::Layout &l) {
        k_l = l.in(logits, (size_t)count * frames_ * kClasses);
        k_m = l.out(masks, (size_t)count * kLocal * frames_);
        k_n = l.out(need, (size_t)count * kLocal);
    });
    if (st != FA_OK) return st;
    std::memcpy(desc.host.data(), sessions, (size_t)count * sizeof(int));
    st = desc.upload((size_t)count * sizeof(int), stream);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(od_embedding_inputs_kernel, count, kThreads, 0, stream,
                       static_cast<const int *>(desc.device.data()), k_l, frames_,
                       masks_in_chunk(frames_, chunk_size), r.min_active, d_bits.data(), k_m, k_n));
    FA_CUDA_TRY(H.finish());
    for (int i = 0; i < count; ++i) table[sessions[i]].pending = true;
    return FA_OK;
}

int Databases::advance(int count, const int *sessions, const float *embeddings, const double *offsets,
                       const Resolved &r, bool device, int64_t *assigned, int32_t *seg_counts, int64_t *seg_ids,
                       float *seg_values) {
    const char *where = "fa_od_advance";
    int st = check_sessions(table, count, sessions, where);
    if (st != FA_OK) return st;
    if (count > 0 && (!embeddings || !offsets || !assigned || !seg_counts || !seg_ids || !seg_values)) {
        set_error("%s: embeddings, offsets, assigned, seg_counts, seg_ids and seg_values must be non-null", where);
        return FA_INVALID_ARGUMENT;
    }
    long long most = 0;
    for (int i = 0; i < count; ++i) {
        if (!table[sessions[i]].pending) {
            set_error("%s: session %d has no staged chunk", where, sessions[i]);
            return FA_INVALID_ARGUMENT;
        }
        if (!std::isfinite(offsets[i])) {
            set_error("%s: chunk offset %d is not finite", where, i);
            return FA_INVALID_ARGUMENT;
        }
        most = std::max(most, table[sessions[i]].meta.count);
    }
    if (count == 0) return FA_OK;
    st = reserve((int)std::min<long long>(most + kLocal, INT32_MAX));
    if (st != FA_OK) return st;
    const long long bound = segment_bound(frames_);
    const size_t off_at = ((size_t)count * sizeof(int) + 255) & ~size_t(255);
    st = desc.reserve(off_at + (size_t)count * sizeof(double));
    if (st == FA_OK) st = h_meta.grow((size_t)count * sizeof(SessionMeta));
    if (st != FA_OK) return st;
    HostStaging H(!device, stream);
    const float *k_e;
    long long *k_a, *k_ids;
    int *k_c;
    float *k_v;
    Segment *made;
    SessionMeta *out_meta;
    st = H.carve(d_io, [&](HostStaging::Layout &l) {
        k_e = l.in(embeddings, (size_t)count * kLocal * kDim);
        k_a = reinterpret_cast<long long *>(l.out(assigned, (size_t)count * kLocal * 2));
        k_c = l.out(seg_counts, (size_t)count);
        k_ids = reinterpret_cast<long long *>(l.out(seg_ids, (size_t)(count * bound * 2)));
        k_v = l.out(seg_values, (size_t)(count * bound * 3));
        made = l.take<Segment>((size_t)(count * bound * 2));
        out_meta = l.take<SessionMeta>((size_t)count);
    });
    if (st != FA_OK) return st;
    char *hd = static_cast<char *>(desc.host.data());
    std::memcpy(hd, sessions, (size_t)count * sizeof(int));
    std::memcpy(hd + off_at, offsets, (size_t)count * sizeof(double));
    st = desc.upload(off_at + (size_t)count * sizeof(double), stream);
    if (st != FA_OK) return st;
    const char *dd = static_cast<const char *>(desc.device.data());
    const long long seq0 = next_seq((long long)count * kLocal);
    AdvanceArgs args{reinterpret_cast<const int *>(dd), k_e, reinterpret_cast<const double *>(dd + off_at),
                     d_db.data(), d_meta.data(), d_bits.data(), made, out_meta, k_a, k_c, k_ids, k_v, capacity_, bound,
                     seq0,
                     frames_, r};
    FA_CUDA_TRY(launch(od_advance_kernel, count, kThreads, 0, stream, args));
    FA_CUDA_TRY(H.back());
    // the headers come back so the next call can size the databases: one synchronisation per tick
    FA_CUDA_TRY(cudaMemcpyAsync(h_meta.data(), out_meta, (size_t)count * sizeof(SessionMeta), cudaMemcpyDeviceToHost,
                                stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    for (int i = 0; i < count; ++i) {
        table[sessions[i]].meta = h_meta.data()[i];
        table[sessions[i]].pending = false;
    }
    return FA_OK;
}

int Databases::query(int session, int count, const float *embeddings, bool device, float *distances) {
    const char *where = "fa_od_query";
    int st = table.check(1, &session, where);
    if (st != FA_OK) return st;
    if (count < 0 || (count > 0 && (!embeddings || !distances))) {
        set_error("%s: count %d must be >= 0 with embeddings and distances non-null", where, count);
        return FA_INVALID_ARGUMENT;
    }
    const long long n = table[session].meta.count;
    if (count == 0 || n == 0) return FA_OK;
    HostStaging H(!device, stream);
    const float *k_q;
    float *k_d;
    st = H.carve(d_io, [&](HostStaging::Layout &l) {
        k_q = l.in(embeddings, (size_t)count * kDim);
        k_d = l.out(distances, (size_t)(count * n));
    });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(od_query_kernel, count, kThreads, 0, stream, d_db.data() + (size_t)session * capacity_, n, k_q,
                       k_d));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int Databases::speaker_count(int session, long long *count, long long *next_id) {
    const int st = table.check(1, &session, "fa_od_speaker_count");
    if (st != FA_OK) return st;
    *count = table[session].meta.count;
    *next_id = table[session].meta.next_id;
    return FA_OK;
}

int Databases::load(int session, std::vector<Speaker> &db) {
    const long long n = table[session].meta.count;
    db.resize((size_t)n);
    if (n)
        FA_CUDA_TRY(cudaMemcpyAsync(db.data(), d_db.data() + (size_t)session * capacity_, (size_t)n * sizeof(Speaker),
                                    cudaMemcpyDeviceToHost, stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    return FA_OK;
}

int Databases::read(int session, SpeakerView *views, float *current, float *raws) {
    int st = table.check(1, &session, "fa_od_read");
    if (st != FA_OK) return st;
    std::vector<Speaker> db;
    st = load(session, db);
    if (st != FA_OK) return st;
    for (size_t i = 0; i < db.size(); ++i) {
        const SpeakerMeta &m = db[i].m;
        if (views)
            views[i] = SpeakerView{m.key, m.numeric, m.update_count, m.duration, m.named, m.has_numeric, m.permanent,
                                   m.raw_count};
        if (current) std::memcpy(current + i * kDim, db[i].current, sizeof(db[i].current));
        if (raws)
            for (int j = 0; j < kFifo; ++j) {
                float *o = raws + (i * kFifo + j) * kDim;
                if (j < m.raw_count) std::memcpy(o, raw_row(db[i], j), kDim * sizeof(float));
                else std::memset(o, 0, kDim * sizeof(float));
            }
    }
    return FA_OK;
}

int Databases::write(int session, const std::vector<Speaker> &db, const SessionMeta &meta) {
    int st = reserve((int)std::min<long long>((long long)db.size(), INT32_MAX));
    if (st != FA_OK) return st;
    if (!db.empty())
        FA_CUDA_TRY(cudaMemcpyAsync(d_db.data() + (size_t)session * capacity_, db.data(), db.size() * sizeof(Speaker),
                                    cudaMemcpyHostToDevice, stream));
    FA_CUDA_TRY(cudaMemcpyAsync(d_meta.data() + session, &meta, sizeof(meta), cudaMemcpyHostToDevice, stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    table[session].meta = meta;
    return FA_OK;
}

// ------------------------------------------------------------------------------------------------ model inputs
int inputs_call(CallContext &C, bool on_device, const float *audio, const int64_t *offsets, int count,
                long long chunk_size, float *segmentation, float *waveform, float *mask, int frames) {
    if (count == 0) return FA_OK;
    const long long total = offsets[count];
    int st = C.stage.reserve((size_t)count * sizeof(InputJob));
    if (st != FA_OK) return st;
    auto *jobs = static_cast<InputJob *>(C.stage.host.data());
    for (int b = 0; b < count; ++b) {
        const long long len = offsets[b + 1] - offsets[b];
        jobs[b] = chunk_size > 0 ? InputJob{offsets[b], std::min(len, chunk_size), chunk_size}
                                 : InputJob{offsets[b], len, len};
    }
    st = C.stage.upload((size_t)count * sizeof(InputJob), C.stream);
    if (st != FA_OK) return st;
    HostStaging H(!on_device, C.stream);
    const float *k_a;
    float *k_s, *k_w, *k_m;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        k_a = l.in(total > 0 ? audio : nullptr, (size_t)total);
        k_s = l.out(segmentation, (size_t)count * kModelSamples);
        k_w = l.out(waveform, (size_t)count * kModelSamples);
        k_m = l.out(mask, (size_t)count * frames);
    });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(od_inputs_kernel, dim3(40, (unsigned)std::min(count, 65535)), dim3(kThreads), 0, C.stream,
                       static_cast<const InputJob *>(C.stage.device.data()), k_a, k_s, k_w, k_m, frames, count));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

} // namespace od
} // namespace fa
