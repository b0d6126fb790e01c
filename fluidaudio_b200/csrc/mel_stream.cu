// Live log-mel streams: SortformerDiarizer's incremental mel stream (SortformerDiarizer.swift:204-217 reset, :417-424
// addAudio, :842-870 emit every covered frame, :876-901 finish with a pre-emphasis-cancelling decay tail) for any number
// of sessions on one MelPlan.
//
// The reference keeps, per session, an audio buffer seeded with nFFT/2 zeros, lastAudioSample, the real samples received
// and the frames emitted.  Each emit runs computeFlatTransposed(.prePadded, expectedFrameCount: count) over the buffer,
// then drops count*hop samples.  Here the buffer's unconsumed samples (the carry) and lastAudioSample live in HBM, one
// fixed slot per session: between pushes a session carries fewer than nFFT/2 + win/2 samples (DESIGN §4.1c), so a slot
// holds round_up4(nFFT/2 + win/2) floats.  The counters live on the host, which therefore knows every frame count before
// anything runs.
//
// One push, whatever the number of sessions:
//   H2D samples (host push) + H2D descriptors -> mel_stream_ingest_kernel (one CTA per session with work) -> one
//   MelPlan launch over the emitting sessions' units (.prePadded, time-major) -> D2H rows + synchronise (host push).
// A host push stages its samples and rows in the plan's staging buffer (HostStaging, fa_common.cuh).
// The ingest CTA assembles [carry | new samples | tail] contiguously at a 16-byte aligned arena offset (the mel kernel's
// bulk-copy path), copies the session's `last` into its MelUnit, then writes back the new carry and `last`.
#include "fa_common.cuh"
#include "mel_plan.h"

#include <algorithm>
#include <cuda_runtime.h>
#include <vector>

namespace fa {
namespace mel {

struct MelStreamJob {
    long long src;      // offset of the pushed samples in the source buffer
    long long n_new;    // pushed samples
    long long arena;    // offset of the session's input [carry | new (| tail)] in the arena, a multiple of 4; -1: no frame
    long long arena2;   // finish after an emit in the same push: offset of [buffer[consumed ..) | tail]; -1 otherwise
    int session;
    int carry_len;      // samples carried in
    int consumed;       // count * hop of the (first) emit
    int tail;           // decay-tail samples appended to the last input (0 or nFFT/2)
    int unit;           // MelUnit of the (first) emit; a split finish's second unit follows it
    int finish;         // the session ends with this push: no carry write-back
};

static constexpr int kIngestThreads = 256;

__global__ void __launch_bounds__(kIngestThreads) mel_stream_ingest_kernel(const MelStreamJob *__restrict__ jobs,
                                                                           const float *__restrict__ src, float *carry_all,
                                                                           float *last_all, float *arena, MelUnit *units,
                                                                           int capacity, float preemph) {
    const MelStreamJob J = jobs[blockIdx.x];
    const int tid = threadIdx.x;
    float *carry = carry_all + (size_t)J.session * capacity;
    const float *x = src + J.src;
    if (J.unit < 0) {   // no frame this push: the samples join the carry (its bound leaves room for them)
        for (long long k = tid; k < J.n_new; k += kIngestThreads) carry[J.carry_len + k] = x[k];
        return;
    }
    const long long L = J.carry_len + J.n_new;
    float *buf = arena + J.arena;
    for (int k = tid; k < J.carry_len; k += kIngestThreads) buf[k] = carry[k];
    for (long long k = tid; k < J.n_new; k += kIngestThreads) buf[J.carry_len + k] = x[k];
    if (tid == 0) units[J.unit].last = last_all[J.session];
    __syncthreads();   // the whole buffer is in the arena: the carry may be overwritten, the split copy read
    const bool split = J.arena2 >= 0;
    const long long left = L - (split ? J.consumed : 0);   // the buffer the finishing emit sees, before its tail
    if (split) {
        float *buf2 = arena + J.arena2;
        for (long long k = tid; k < left; k += kIngestThreads) buf2[k] = buf[J.consumed + k];
        if (tid == 0) units[J.unit + 1].last = buf[J.consumed - 1];
    }
    if (J.tail && tid == 0) {
        // padAndEmitRemainingMelLocked (:888-896): value = buffer.last, value *= preemph per sample, float32 rounded at
        // every step; zeros when preemph is 0 or the buffer is empty
        float *t = (split ? arena + J.arena2 : buf) + left;
        const bool decay = preemph != 0.0f && left > 0;
        float v = left > 0 ? buf[L - 1] : 0.0f;
        for (int i = 0; i < J.tail; ++i) {
            v = decay ? __fmul_rn(v, preemph) : 0.0f;
            t[i] = v;
        }
    }
    if (!J.finish) {   // emitMelFramesLocked (:862-865): lastAudioSample = buffer[consumed - 1], drop `consumed` samples
        for (long long k = tid; k < L - J.consumed; k += kIngestThreads) carry[k] = buf[J.consumed + k];
        if (tid == 0) last_all[J.session] = buf[J.consumed - 1];
    }
}

static inline long long round_up4(long long v) { return (v + 3) & ~3LL; }

// Frames of one push: `first` from addAudio's preprocessAudioToFeaturesLocked (:847-854), `second` from
// padAndEmitRemainingMelLocked (:876-883) when the push finishes the session.  Integer division truncates like Swift's.
static void push_frames(const MelConfig &c, const MelSession &m, long long n, bool fin, long long &first, long long &second) {
    first = second = 0;
    if (m.finished) return;   // shouldDropAudioLocked
    const long long r = m.received + n, half_win = c.win_length / 2;
    if (r >= half_win) first = std::max(0LL, (r - half_win) / c.hop_length + 1 - m.emitted);
    if (fin && r > 0) second = std::max(0LL, 1 + (r + c.n_fft - c.win_length) / c.hop_length - m.emitted - first);
}

int MelStreamSet::check_config(const MelConfig &c) {
    if (!c.neutral()) {
        fa::set_error("mel stream: live streams run AudioMelSpectrogram only, not a handle with fa_mel_ex_config fields set");
        return FA_INVALID_ARGUMENT;
    }
    if (c.pad_to > 1) {
        fa::set_error("mel stream: pad_to must be 0 or 1 (an emit returns exactly its frames), got %d", c.pad_to);
        return FA_INVALID_ARGUMENT;
    }
    if (c.hop_length > c.win_length) {
        fa::set_error("mel stream: hop_length (%d) must not exceed win_length (%d)", c.hop_length, c.win_length);
        return FA_INVALID_ARGUMENT;
    }
    return FA_OK;
}

int MelStreamSet::open(MelPlan &p, int *session) {
    int st = check_config(p.cfg);
    if (st != FA_OK) return st;
    const int half = p.cfg.n_fft / 2;
    capacity = (int)round_up4(half + p.cfg.win_length / 2);
    cudaStream_t s = p.streams[1];
    auto grow = [&](int grown) { return grow_slots(table.slots(), grown, s, d_carry, capacity, d_last, 1); };
    // resetMelStreamLocked (:204-217): the buffer is nFFT/2 zeros, lastAudioSample 0, counters cleared
    auto init = [&](int id) -> int {
        FA_CUDA_TRY(cudaMemsetAsync(d_carry.data() + (size_t)id * capacity, 0, (size_t)half * sizeof(float), s));
        FA_CUDA_TRY(cudaMemsetAsync(d_last.data() + id, 0, sizeof(float), s));
        table[id].carry_len = half;
        return FA_OK;
    };
    return table.open(64, grow, init, session);
}

int MelStreamSet::close(int session) { return table.close(session, "mel stream"); }

long long MelStreamSet::frames(const MelPlan &p, int session, long long n, bool finish) const {
    if (!table.valid(session) || n < 0) return -1;
    long long first, second;
    push_frames(p.cfg, table[session], n, finish, first, second);
    return first + second;
}

int MelStreamSet::push(MelPlan &p, int count, const int *sessions, const float *audio, const int64_t *offsets,
                       const int *finish, bool device, float *out, long long out_len, int64_t *frames_out) {
    const MelConfig &c = p.cfg;
    const int M = c.n_mels, hop = c.hop_length, half = c.n_fft / 2;
    if (count < 0 || (count > 0 && (!sessions || !offsets || !frames_out))) {
        fa::set_error("mel stream push: count must be >= 0, sessions / offsets / frames non-null");
        return FA_INVALID_ARGUMENT;
    }
    if (count == 0) return FA_OK;
    if (offsets[0] < 0) {
        fa::set_error("mel stream push: offsets[0] is negative (%lld)", (long long)offsets[0]);
        return FA_INVALID_ARGUMENT;
    }
    int st = table.check(count, sessions, "mel stream push");
    if (st != FA_OK) return st;
    for (int i = 0; i < count; ++i)
        if (offsets[i + 1] < offsets[i]) {
            fa::set_error("mel stream push: offsets decrease at %d (%lld > %lld)", i, (long long)offsets[i],
                          (long long)offsets[i + 1]);
            return FA_INVALID_ARGUMENT;
        }
    const long long total_new = offsets[count] - offsets[0];
    if (total_new > 0 && !audio) {
        fa::set_error("mel stream push: audio is null");
        return FA_INVALID_ARGUMENT;
    }
    struct Step {
        long long first, second, L;
        bool fin;
    };
    std::vector<Step> step(count);
    std::vector<MelSession> next(count);
    long long rows = 0, arena = 0;
    int units = 0, jobs = 0;
    const long long bound = half + c.win_length / 2;   // carried samples stay below this (DESIGN §4.1c)
    for (int i = 0; i < count; ++i) {
        const int id = sessions[i];
        const MelSession &m = table[id];
        Step &S = step[i];
        const long long n = offsets[i + 1] - offsets[i];
        S.fin = finish && finish[i];
        push_frames(c, m, n, S.fin, S.first, S.second);
        S.L = m.carry_len + n;
        rows += S.first + S.second;
        const long long consumed = S.first * hop, tail = S.second ? half : 0;
        next[i] = m.finished ? m : MelSession{S.L - consumed, m.received + n, m.emitted + S.first + S.second, S.fin};
        if (m.finished) continue;
        if (consumed > S.L || (!S.fin && S.L - consumed >= bound)) {
            fa::set_error("internal: mel stream carry bound (session %d: %lld samples, %lld consumed)", id, S.L, consumed);
            return FA_RUNTIME_ERROR;
        }
        if (S.first + S.second == 0) {
            if (n > 0 && !S.fin) ++jobs;   // samples join the carry
            continue;
        }
        ++jobs;
        const bool split = S.first > 0 && S.second > 0;
        units += split ? 2 : 1;
        arena += round_up4(S.L + (split ? 0 : tail)) + (split ? round_up4(S.L - consumed + tail) : 0);
    }
    if (rows > 0 && (!out || out_len < rows * M)) {
        fa::set_error("mel stream push: output needs %lld floats, buffer has %lld", rows * M, out ? out_len : 0);
        return FA_OUTPUT_TOO_SMALL;
    }

    // ---- buffers: the pushed samples, from offsets[0] on, and the rows
    cudaStream_t s = p.streams[1];
    HostStaging H(!device, s);
    const float *src;
    float *k_out;
    const size_t units_bytes = (((size_t)units * sizeof(MelUnit)) + 15) & ~size_t(15);
    const size_t desc_bytes = units_bytes + (size_t)jobs * sizeof(MelStreamJob);
    st = desc.reserve(std::max<size_t>(desc_bytes, 4096));
    if (st == FA_OK) st = d_arena.grow((size_t)std::max(arena, 1024LL) * sizeof(float));
    if (st == FA_OK)
        st = H.carve(p.staging, [&](HostStaging::Layout &l) {
            src = l.in(audio ? audio + offsets[0] : nullptr, (size_t)total_new, 8);
            k_out = l.out(out, (size_t)(rows * M));
        });
    if (st != FA_OK) return st;

    // ---- descriptors: units, then jobs
    MelUnit *hu = static_cast<MelUnit *>(desc.host.data());
    MelStreamJob *hj = reinterpret_cast<MelStreamJob *>(static_cast<char *>(desc.host.data()) + units_bytes);
    MelUnit *du = static_cast<MelUnit *>(desc.device.data());
    MelStreamJob *dj = reinterpret_cast<MelStreamJob *>(static_cast<char *>(desc.device.data()) + units_bytes);
    long long row = 0, a = 0;
    int u = 0, j = 0;
    for (int i = 0; i < count; ++i) {
        const int id = sessions[i];
        const Step &S = step[i];
        const long long n = offsets[i + 1] - offsets[i], emit = S.first + S.second;
        if (table[id].finished || (emit == 0 && (n == 0 || S.fin))) continue;
        MelStreamJob &J = hj[j++];
        J = MelStreamJob{offsets[i] - offsets[0], n, -1, -1, id, (int)table[id].carry_len, 0, 0, -1, S.fin ? 1 : 0};
        if (emit == 0) continue;
        const bool split = S.first > 0 && S.second > 0;
        J.consumed = (int)(S.first * hop);
        J.tail = S.second ? half : 0;
        J.unit = u;
        J.arena = a;
        const long long c1 = split ? S.first : emit;   // frames of the first unit
        const long long n1 = S.L + (split ? 0 : J.tail);
        hu[u++] = MelUnit{a, n1, row * M, c1, 0, c1, 0.0f, 0};   // .last: written by the ingest kernel
        a += round_up4(n1);
        if (split) {
            J.arena2 = a;
            const long long n2 = S.L - J.consumed + J.tail;
            hu[u++] = MelUnit{a, n2, (row + c1) * M, S.second, 0, S.second, 0.0f, 0};
            a += round_up4(n2);
        }
        row += emit;
    }
    number_tiles(hu, units);

    // ---- device work, all on the compute stream
    if (desc_bytes) {
        st = desc.upload(desc_bytes, s);
        if (st != FA_OK) return st;
    }
    if (jobs) {
        FA_CUDA_TRY(fa::launch(mel_stream_ingest_kernel, jobs, kIngestThreads, 0, s, dj, src, d_carry.data(), d_last.data(),
                               d_arena.data(), du, capacity, c.preemph));
    }
    if (units) {
        // `last` lives in the device units (written by the ingest kernel): the launch reads them from HBM, never inline
        st = p.launch(du, hu, units, false, d_arena.data(), k_out, FA_MEL_PAD_PREPADDED, FA_MEL_TIME_MAJOR, s);
        if (st != FA_OK) return st;
    }
    FA_CUDA_TRY(H.finish());

    table.commit(count, sessions, next.data());
    for (int i = 0; i < count; ++i) frames_out[i] = step[i].first + step[i].second;
    return FA_OK;
}

} // namespace mel
} // namespace fa
