// LS-EEND live feature streams: LSEENDFeatureProvider (Diarizer/LS-EEND/LSEENDPreprocessor.swift:46-384) for any number
// of sessions on one MelPlan.
//
// The provider keeps two StreamingChunkQueues (:284-384), the running mean (cmnMean, cmnCount) and decoderMaskEnd.  Here
// each session owns one fixed slot in HBM: its unread audio (fewer than chunkSamples + nFFT - hop samples), its unread
// mel rows (fewer than melFrames), cmnMean, and one snapshot copy of all three.  The host mirrors the lengths, cmnCount,
// decoderMaskEnd and whether a snapshot exists (lseend_plan.h), so it knows every count before anything runs.
//
// A push is enqueueAudio, drainRightContextWithSilence when asked, and emitNextChunk until none is ready (the caller's
// flow, LSEENDDiarizer.swift:119-157, 233-268).  processAudioQueue runs once over the samples and the drain together:
// popAllChunks pops the same frames either way, the drain's shortfall depends only on the unread count modulo whole
// chunks, and every frame's log-mel depends on its own window alone.  Four launches whatever the session count:
//   lseend_ingest_kernel   one CTA per session with samples: [carry | new | drain zeros] at a 16-byte aligned arena
//                          offset, the session's mel rows in front of the room for its new ones, the new audio carry
//                          back to the slot (a session that completes no audio chunk only appends to its carry)
//   MelPlan::launch        every emitting session's popAllChunks slice, .prePadded, time-major, into its mel queue
//   lseend_cmn_kernel      one thread per (session, mel) down the new rows in order: log10 scaling and the running mean
//   lseend_gather_kernel   one CTA per emitting session: its model-input chunks, mask windows and warm-up counts, then
//                          the mel rows left unread back to the slot
// A push in which no session completes an audio chunk issues the ingest launch alone (none at all without samples).
#include "lseend_streams.h"

#include <algorithm>
#include <cmath>
#include <cuda_runtime.h>
#include <vector>

namespace fa {
namespace lseend {

struct Job {
    long long src;        // offset of the pushed samples in the source buffer
    long long n_new;      // pushed samples
    long long zeros;      // drain zeros after them
    long long arena;      // offset of [carry | new | zeros] in the arena; -1: no audio chunk completes
    long long queue;      // offset of the mel queue [carried rows | new rows] in the arena
    long long out_chunk;  // first output chunk of the session
    long long cmn_count;  // frames seen before this push
    int session;
    int carry;            // audio samples carried in
    int consumed;         // samples popAllChunks drops
    int rows;             // mel rows carried in
    int frames;           // mel rows computed
    int chunks;           // chunks emitted
    int mask_end;         // decoderMaskEnd before the push
};

struct Shape {
    int half, mel_off, mean_half, n_mels, mel_frames, chunk_mels, chunk_size, conv_delay, mask_length;
};

static constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads) lseend_ingest_kernel(const Job *__restrict__ jobs, const float *__restrict__ src,
                                                                 float *state, float *arena, Shape S) {
    const Job J = jobs[blockIdx.x];
    const int tid = threadIdx.x;
    float *carry = state + (size_t)J.session * 2 * S.half;
    const float *x = src + J.src;
    if (J.arena < 0) {   // no chunk completes: the samples and the zeros join the carry (its bound leaves room)
        for (long long k = tid; k < J.n_new; k += kThreads) carry[J.carry + k] = x[k];
        for (long long k = tid; k < J.zeros; k += kThreads) carry[J.carry + J.n_new + k] = 0.0f;
        return;
    }
    float *buf = arena + J.arena;
    const long long L = J.carry + J.n_new + J.zeros;
    for (int k = tid; k < J.carry; k += kThreads) buf[k] = carry[k];
    for (long long k = tid; k < J.n_new; k += kThreads) buf[J.carry + k] = x[k];
    for (long long k = tid; k < J.zeros; k += kThreads) buf[J.carry + J.n_new + k] = 0.0f;
    const float *mel = carry + S.mel_off;
    float *q = arena + J.queue;
    for (long long k = tid; k < (long long)J.rows * S.n_mels; k += kThreads) q[k] = mel[k];
    __syncthreads();   // the whole input is in the arena: the carry may be overwritten
    for (long long k = tid; k < L - J.consumed; k += kThreads) carry[k] = buf[J.consumed + k];
}

__global__ void lseend_cmn_kernel(const Job *__restrict__ jobs, float *arena, float *means, Shape S, float scale) {
    const Job J = jobs[blockIdx.x];
    const int m = blockIdx.y * blockDim.x + threadIdx.x;
    if (m >= S.n_mels) return;
    float *mean = means + (size_t)J.session * 2 * S.mean_half + m;
    float *x = arena + J.queue + (long long)J.rows * S.n_mels;
    *mean = scale_cmn_column(x, J.frames, S.n_mels, m, *mean, J.cmn_count, scale);
}

__global__ void __launch_bounds__(kThreads) lseend_gather_kernel(const Job *__restrict__ jobs, const float *arena,
                                                                 float *state, float *features, float *masks,
                                                                 int *warmup, Shape S) {
    const Job J = jobs[blockIdx.x];
    const int tid = threadIdx.x, M = S.n_mels;
    const float *q = arena + J.queue;
    const long long chunk_floats = (long long)S.mel_frames * M, step = (long long)S.chunk_mels * M;
    for (int j = 0; j < J.chunks; ++j) {   // popNextChunk: rows [j * chunk_mels, j * chunk_mels + mel_frames)
        float *out = features + (J.out_chunk + j) * chunk_floats;
        const float *in = q + j * step;
        for (long long k = tid; k < chunk_floats; k += kThreads) out[k] = in[k];
    }
    for (int k = tid; k < J.chunks * S.chunk_size; k += kThreads) {
        const int j = k / S.chunk_size, t = k - j * S.chunk_size;
        const int end = min(J.mask_end + (j + 1) * S.chunk_size, S.mask_length);
        masks[(J.out_chunk + j) * S.chunk_size + t] = mask_value(end, S.chunk_size, S.conv_delay, t);
        if (t == 0) warmup[J.out_chunk + j] = warmup_frames(end, S.chunk_size, S.mask_length);
    }
    float *mel = state + (size_t)J.session * 2 * S.half + S.mel_off;
    const long long left = ((long long)J.rows + J.frames - (long long)J.chunks * S.chunk_mels) * M;
    const float *rest = q + J.chunks * step;
    for (long long k = tid; k < left; k += kThreads) mel[k] = rest[k];
}

// kind 0: snapshot (live -> copy), 1: rollback (copy -> live), 2: reset (live zeroed: nFFT/2 zero samples, context_size
// zero rows and a zero mean, the lengths being the host's)
__global__ void __launch_bounds__(kThreads) lseend_slot_kernel(const int *__restrict__ ids, float *state, float *means,
                                                               Shape S, int kind) {
    const size_t id = ids[blockIdx.x];
    float *live = state + id * 2 * S.half, *copy = live + S.half;
    float *mlive = means + id * 2 * S.mean_half, *mcopy = mlive + S.mean_half;
    for (int k = threadIdx.x; k < S.half; k += kThreads) {
        if (kind == 0) copy[k] = live[k];
        else live[k] = kind == 1 ? copy[k] : 0.0f;
    }
    for (int k = threadIdx.x; k < S.mean_half; k += kThreads) {
        if (kind == 0) mcopy[k] = mlive[k];
        else mlive[k] = kind == 1 ? mcopy[k] : 0.0f;
    }
}

static inline long long round_up4(long long v) { return (v + 3) & ~3LL; }

int StreamSet::init(const Config &c) {
    int st = resolve(c, sz);
    if (st != FA_OK) return st;
    cfg = c;
    // the provider's AudioMelSpectrogram (:70-81): preemph 0, padTo 0, logFloor 1e-10 clamped, periodic Hann
    mel::MelConfig m{};
    m.sample_rate = c.sample_rate;
    m.n_mels = c.n_mels;
    m.n_fft = sz.n_fft;
    m.hop_length = c.hop_length;
    m.win_length = c.win_length;
    m.preemph = 0.0f;
    m.pad_to = 0;
    m.log_floor = 1e-10f;
    m.log_floor_mode = 1;
    m.window_periodic = 1;
    st = plan.init(m);
    if (st != FA_OK) return st;
    plan.precision = c.precision;
    mel_off = (int)round_up4(sz.audio_capacity);
    half = mel_off + (int)round_up4((long long)sz.mel_frames * c.n_mels);
    mean_half = (int)round_up4(c.n_mels);
    return FA_OK;
}

int StreamSet::open(int *session) {
    cudaStream_t s = plan.streams[1];
    auto grow = [&](int grown) { return grow_slots(table.slots(), grown, s, d_state, 2 * (size_t)half, d_mean, 2 * (size_t)mean_half); };
    auto init = [&](int id) -> int {   // :94-109
        FA_CUDA_TRY(cudaMemsetAsync(d_state.data() + (size_t)id * 2 * half, 0, (size_t)half * sizeof(float), s));
        FA_CUDA_TRY(cudaMemsetAsync(d_mean.data() + (size_t)id * 2 * mean_half, 0, (size_t)mean_half * sizeof(float), s));
        table[id].now = fresh(cfg, sz);
        return FA_OK;
    };
    return table.open(64, grow, init, session);
}

int StreamSet::close(int session) { return table.close(session, "lseend stream"); }

// A push carries at most this many samples per session, so every count the planning forms fits comfortably in int64.
static constexpr long long kMaxPushSamples = 1LL << 40;

long long StreamSet::chunks(int session, long long n, bool drain) const {
    if (!table.valid(session) || n < 0 || n > kMaxPushSamples) return -1;
    return plan_push(cfg, sz, table[session].now, n, drain).chunks;
}

int StreamSet::push(int count, const int *sessions, const float *audio, const int64_t *offsets, const int *drain,
                    bool device, float *features, long long features_len, float *masks, long long masks_len,
                    int *warmup, long long warmup_len, int64_t *chunks_out) {
    const int M = cfg.n_mels;
    if (count < 0 || (count > 0 && (!sessions || !offsets || !chunks_out))) {
        set_error("lseend stream push: count must be >= 0, sessions / offsets / chunks non-null");
        return FA_INVALID_ARGUMENT;
    }
    if (count == 0) return FA_OK;
    if (offsets[0] < 0) {
        set_error("lseend stream push: offsets[0] is negative (%lld)", (long long)offsets[0]);
        return FA_INVALID_ARGUMENT;
    }
    int st = table.check(count, sessions, "lseend stream push");
    if (st != FA_OK) return st;
    for (int i = 0; i < count; ++i)
        if (offsets[i + 1] < offsets[i] || offsets[i + 1] - offsets[i] > kMaxPushSamples) {
            set_error("lseend stream push: offsets decrease at %d, or a session gets more than 2^40 samples (%lld, %lld)",
                      i, (long long)offsets[i], (long long)offsets[i + 1]);
            return FA_INVALID_ARGUMENT;
        }
    const long long total_new = offsets[count] - offsets[0];
    if (total_new > 0 && !audio) {
        set_error("lseend stream push: audio is null");
        return FA_INVALID_ARGUMENT;
    }
    std::vector<Step> step(count);
    long long total_chunks = 0, arena = 0;
    int jobs = 0, emitting = 0, units = 0;
    for (int i = 0; i < count; ++i) {
        const Lengths &m = table[sessions[i]].now;
        Step &t = step[i];
        t = plan_push(cfg, sz, m, offsets[i + 1] - offsets[i], drain && drain[i]);
        if (t.next.audio >= sz.audio_capacity || t.next.mel >= sz.mel_frames || t.next.mel < 0) {
            set_error("internal: lseend stream carry bound (session %d: %lld samples, %lld rows)", sessions[i],
                      t.next.audio, t.next.mel);
            return FA_RUNTIME_ERROR;
        }
        total_chunks += t.chunks;
        if (t.frames > 0) {
            ++emitting;
            ++units;
            arena += round_up4(t.unread) + round_up4((m.mel + t.frames) * M);
        }
        if (t.unread > m.audio) ++jobs;   // samples or drain zeros arrive
    }
    if (total_chunks > 0 && (!features || features_len < total_chunks * sz.mel_frames * M || !masks ||
                             masks_len < total_chunks * cfg.chunk_size || !warmup || warmup_len < total_chunks)) {
        set_error("lseend stream push: the outputs need %lld feature floats, %lld mask floats and %lld warm-up counts, "
                  "have %lld, %lld and %lld",
                  total_chunks * sz.mel_frames * M, total_chunks * cfg.chunk_size, total_chunks,
                  features ? features_len : 0, masks ? masks_len : 0, warmup ? warmup_len : 0);
        return FA_INVALID_ARGUMENT;
    }

    // ---- buffers: the pushed samples from offsets[0] on, and the three outputs
    cudaStream_t s = plan.streams[1];
    HostStaging H(!device, s);
    const float *src = nullptr;
    float *k_feat = nullptr, *k_mask = nullptr;
    int *k_warm = nullptr;
    const size_t units_bytes = (((size_t)units * sizeof(mel::MelUnit)) + 15) & ~size_t(15);
    const size_t desc_bytes = units_bytes + (size_t)jobs * sizeof(Job);
    st = desc.reserve(std::max<size_t>(desc_bytes, 4096));
    if (st == FA_OK) st = d_arena.grow((size_t)std::max(arena, 1024LL) * sizeof(float));
    if (st == FA_OK)
        st = H.carve(plan.staging, [&](HostStaging::Layout &l) {
            src = l.in(audio ? audio + offsets[0] : nullptr, (size_t)total_new, 8);
            k_feat = l.out(total_chunks ? features : nullptr, (size_t)(total_chunks * sz.mel_frames * M));
            k_mask = l.out(total_chunks ? masks : nullptr, (size_t)(total_chunks * cfg.chunk_size));
            k_warm = l.out(total_chunks ? warmup : nullptr, (size_t)total_chunks);
        });
    if (st != FA_OK) return st;

    // ---- descriptors: units, then jobs, the emitting ones first (the cmn and gather launches cover those alone)
    mel::MelUnit *hu = static_cast<mel::MelUnit *>(desc.host.data());
    Job *hj = reinterpret_cast<Job *>(static_cast<char *>(desc.host.data()) + units_bytes);
    mel::MelUnit *du = static_cast<mel::MelUnit *>(desc.device.data());
    Job *dj = reinterpret_cast<Job *>(static_cast<char *>(desc.device.data()) + units_bytes);
    long long a = 0, chunk = 0;
    int u = 0, j = 0;
    for (int pass = 0; pass < 2; ++pass)
        for (int i = 0; i < count; ++i) {
            const Step &t = step[i];
            const Lengths &m = table[sessions[i]].now;
            if ((t.frames > 0) != (pass == 0) || t.unread == m.audio) continue;
            Job &J = hj[j++];
            J = Job{offsets[i] - offsets[0], offsets[i + 1] - offsets[i], t.zeros, -1, 0, 0, m.cmn_count, sessions[i],
                    (int)m.audio, (int)t.consumed, (int)m.mel, (int)t.frames, (int)t.chunks, m.mask_end};
            if (t.frames == 0) continue;
            J.arena = a;
            J.queue = a + round_up4(t.unread);
            J.out_chunk = chunk;
            // the popAllChunks slice [0, consumed + nFFT - hop) of the assembled queue (:372-373)
            const long long L = t.consumed + sz.audio_context;
            hu[u++] = mel::MelUnit{J.arena, L, J.queue + m.mel * M, t.frames, 0, t.frames, 0.0f, 0};
            a = J.queue + round_up4((m.mel + t.frames) * M);
            chunk += t.chunks;
        }
    mel::number_tiles(hu, units);

    // ---- device work, all on the compute stream
    const Shape S{half, mel_off, mean_half, M, sz.mel_frames, sz.chunk_mels, cfg.chunk_size, cfg.conv_delay,
                  sz.mask_length};
    if (desc_bytes) {
        st = desc.upload(desc_bytes, s);
        if (st != FA_OK) return st;
    }
    if (jobs) FA_CUDA_TRY(fa::launch(lseend_ingest_kernel, jobs, kThreads, 0, s, dj, src, d_state.data(), d_arena.data(), S));
    if (emitting) {
        st = plan.launch(du, hu, units, false, d_arena.data(), d_arena.data(), FA_MEL_PAD_PREPADDED, FA_MEL_TIME_MAJOR, s);
        if (st != FA_OK) return st;
        const float scale = 1.0f / logf(10.0f);   // LSEENDPreprocessor.swift:36, Float arithmetic
        FA_CUDA_TRY(fa::launch(lseend_cmn_kernel, dim3(emitting, (M + 127) / 128), 128, 0, s, dj, d_arena.data(),
                               d_mean.data(), S, scale));
        FA_CUDA_TRY(fa::launch(lseend_gather_kernel, emitting, kThreads, 0, s, dj, d_arena.data(), d_state.data(), k_feat,
                               k_mask, k_warm, S));
    }
    FA_CUDA_TRY(H.finish());

    for (int i = 0; i < count; ++i) {
        table[sessions[i]].now = step[i].next;
        chunks_out[i] = step[i].chunks;
    }
    return FA_OK;
}

int StreamSet::slots(int kind, int count, const int *sessions, const char *where) {
    if (count < 0 || (count > 0 && !sessions)) {
        set_error("%s: count must be >= 0 and sessions non-null", where);
        return FA_INVALID_ARGUMENT;
    }
    int st = table.check(count, sessions, where);
    if (st != FA_OK) return st;
    if (kind == 1)
        for (int i = 0; i < count; ++i)
            if (!table[sessions[i]].has_snapshot) {
                set_error("%s: session %d has no snapshot", where, sessions[i]);
                return FA_INVALID_ARGUMENT;
            }
    if (count == 0) return FA_OK;
    cudaStream_t s = plan.streams[1];
    const size_t bytes = (size_t)count * sizeof(int);
    st = desc.reserve(std::max<size_t>(bytes, 4096));
    if (st != FA_OK) return st;
    std::copy(sessions, sessions + count, static_cast<int *>(desc.host.data()));
    st = desc.upload(bytes, s);
    if (st != FA_OK) return st;
    const Shape S{half, mel_off, mean_half, cfg.n_mels, sz.mel_frames, sz.chunk_mels, cfg.chunk_size, cfg.conv_delay,
                  sz.mask_length};
    FA_CUDA_TRY(fa::launch(lseend_slot_kernel, count, kThreads, 0, s, static_cast<const int *>(desc.device.data()),
                           d_state.data(), d_mean.data(), S, kind));
    for (int i = 0; i < count; ++i) {
        Session &m = table[sessions[i]];
        if (kind == 0) {
            m.snap = m.now;
            m.has_snapshot = true;
        } else {
            m.now = kind == 1 ? m.snap : fresh(cfg, sz);
        }
    }
    return FA_OK;
}

int StreamSet::snapshot(int count, const int *sessions) { return slots(0, count, sessions, "lseend stream snapshot"); }
int StreamSet::rollback(int count, const int *sessions) { return slots(1, count, sessions, "lseend stream rollback"); }
int StreamSet::reset(int count, const int *sessions) { return slots(2, count, sessions, "lseend stream reset"); }

int StreamSet::state(int session, SessionInfo *info, float *audio, float *mel, float *cmn_mean) {
    int st = table.check(1, &session, "lseend stream state");
    if (st != FA_OK) return st;
    const Session &m = table[session];
    cudaStream_t s = plan.streams[1];
    const float *live = d_state.data() + (size_t)session * 2 * half;
    if (audio && m.now.audio)
        FA_CUDA_TRY(cudaMemcpyAsync(audio, live, (size_t)m.now.audio * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (mel && m.now.mel)
        FA_CUDA_TRY(cudaMemcpyAsync(mel, live + mel_off, (size_t)m.now.mel * cfg.n_mels * sizeof(float),
                                    cudaMemcpyDeviceToHost, s));
    if (cmn_mean)
        FA_CUDA_TRY(cudaMemcpyAsync(cmn_mean, d_mean.data() + (size_t)session * 2 * mean_half,
                                    (size_t)cfg.n_mels * sizeof(float), cudaMemcpyDeviceToHost, s));
    FA_CUDA_TRY(cudaStreamSynchronize(s));
    *info = SessionInfo{m.now.audio, m.now.mel, m.now.cmn_count, m.now.mask_end, m.has_snapshot ? 1 : 0};
    return FA_OK;
}

} // namespace lseend
} // namespace fa
