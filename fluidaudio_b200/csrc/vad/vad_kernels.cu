// Voice activity detection on the GPU (vad.h, vad_core.cuh).
//
// Silero live sessions: each session owns one slot in HBM (context, hidden, cell and the pending context as floats;
// processedSamples, triggered, tempEndSample and the pending chunk's sample count as int64).  The host mirrors only
// whether a chunk is pending, which is all a call needs to check before anything runs.  One launch per call:
//   vad_model_inputs_kernel  one CTA per session: [context | processed chunk] into the model input row, the LSTM
//                            state out, the processed chunk's last 64 samples and its sample count into the slot's
//                            pending fields
//   vad_advance_kernel       one CTA per session: the new LSTM state and the pending context into the slot, then
//                            streamingStateMachine on one thread
// Clip calls (fa_vad_segment, fa_fsmn_vad_decide): one thread per clip runs the whole sequential state machine into
// scratch sized by the proven bound (P pairs for P Silero probabilities, (T + 1) / 2 for T FSMN frames), the counts
// come back at the one synchronisation, then one CTA per clip gathers its pairs to their compact place.
#include "vad.h"

#include <algorithm>
#include <cstring>
#include <cuda_runtime.h>
#include <vector>

namespace fa {
namespace vad {

namespace {

constexpr int kThreads = 256;

struct InputJob {
    long long src, n;   // the chunk's offset in the call's audio and its sample count
    int slot;
};

__global__ void __launch_bounds__(kThreads)
    vad_model_inputs_kernel(const InputJob *__restrict__ jobs, const float *__restrict__ audio, float *state,
                            long long *meta, float *__restrict__ audio_input, float *__restrict__ hidden,
                            float *__restrict__ cell) {
    const InputJob J = jobs[blockIdx.x];
    float *S = state + (size_t)J.slot * kSlotFloats;
    const float *x = audio + J.src;
    float *row = audio_input + (size_t)blockIdx.x * kModelInput;
    for (int k = threadIdx.x; k < kModelInput; k += kThreads) {
        const float v = k < kContext ? S[k] : chunk_sample(x, J.n, k - kContext);
        row[k] = v;
        if (k >= kModelInput - kContext) S[kPendingAt + k - (kModelInput - kContext)] = v;
    }
    for (int k = threadIdx.x; k < kState; k += kThreads) {
        hidden[(size_t)blockIdx.x * kState + k] = S[kHiddenAt + k];
        cell[(size_t)blockIdx.x * kState + k] = S[kCellAt + k];
    }
    if (threadIdx.x == 0) meta[(size_t)J.slot * kSlotFields + kPendingCount] = J.n;
}

__global__ void __launch_bounds__(kState)
    vad_advance_kernel(const int *__restrict__ slots, const float *__restrict__ probability,
                       const float *__restrict__ new_hidden, const float *__restrict__ new_cell, float *state,
                       long long *meta, long long *__restrict__ events, Resolved r) {
    const int b = blockIdx.x, k = threadIdx.x;
    float *S = state + (size_t)slots[b] * kSlotFloats;
    S[kHiddenAt + k] = new_hidden[(size_t)b * kState + k];
    S[kCellAt + k] = new_cell[(size_t)b * kState + k];
    if (k < kContext) S[k] = S[kPendingAt + k];
    if (k == 0) {
        long long *m = meta + (size_t)slots[b] * kSlotFields;
        StreamState s{m[kProcessed], m[kTempEnd], m[kTriggered]};
        long long sample;
        const int kind = stream_step(s, probability[b], m[kPendingCount], r, &sample);
        m[kProcessed] = s.processed;
        m[kTempEnd] = s.temp_end;
        m[kTriggered] = s.triggered;
        m[kPendingCount] = -1;
        events[2 * b] = kind;
        events[2 * b + 1] = sample;
    }
}

struct ClipDesc {
    long long in, n;      // the clip's first input row and its row count
    long long scratch;    // its first scratch pair
    long long samples;    // totalSamples (Silero)
};

__global__ void vad_clip_kernel(const ClipDesc *__restrict__ clips, int count, const float *__restrict__ input,
                                int fsmn, Resolved r, long long *scratch, long long *__restrict__ counts) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= count) return;
    const ClipDesc c = clips[b];
    counts[b] = fsmn ? fsmn_clip(input + c.in, c.n, scratch + 2 * c.scratch)
                     : segment_clip(input + c.in, c.n, c.samples, r, scratch + 2 * c.scratch);
}

__global__ void __launch_bounds__(kThreads)
    vad_gather_kernel(const ClipDesc *__restrict__ clips, const long long *__restrict__ counts,
                      const long long *__restrict__ out_at, const long long *__restrict__ scratch,
                      long long *__restrict__ out) {
    const int b = blockIdx.x;
    const long long *src = scratch + 2 * clips[b].scratch;
    long long *dst = out + 2 * out_at[b];
    for (long long k = threadIdx.x; k < 2 * counts[b]; k += kThreads) dst[k] = src[k];
}

} // namespace

// ------------------------------------------------------------------------------------------------ sessions
int StreamSet::init() { return stream.create(); }

int StreamSet::open(int *session) {
    auto grow = [&](int grown) {
        return grow_slots(table.slots(), grown, stream, d_state, (size_t)kSlotFloats, d_meta, (size_t)kSlotFields);
    };
    auto init = [&](int id) -> int {   // VadStreamState.initial(): zero state, tempEndSample nil, nothing pending
        long long *m = d_meta.data() + (size_t)id * kSlotFields;
        FA_CUDA_TRY(cudaMemsetAsync(d_state.data() + (size_t)id * kSlotFloats, 0, kSlotFloats * sizeof(float), stream));
        FA_CUDA_TRY(cudaMemsetAsync(m, 0, 2 * sizeof(long long), stream));
        FA_CUDA_TRY(cudaMemsetAsync(m + kTempEnd, 0xff, 2 * sizeof(long long), stream));
        return FA_OK;
    };
    return table.open(64, grow, init, session);
}

int StreamSet::close(int session) { return table.close(session, "vad stream close"); }

static int check_sessions(const SessionTable<Mirror> &table, int count, const int *sessions, const char *where) {
    if (count < 0 || (count > 0 && !sessions)) {
        set_error("%s: count %d must be >= 0 and sessions non-null", where, count);
        return FA_INVALID_ARGUMENT;
    }
    return table.check(count, sessions, where);
}

int StreamSet::model_inputs(int count, const int *sessions, const float *audio, const int64_t *offsets, bool device,
                            float *audio_input, float *hidden, float *cell) {
    const char *where = "fa_vad_stream_model_inputs";
    int st = check_sessions(table, count, sessions, where);
    if (st != FA_OK) return st;
    if (count > 0 && (!offsets || !audio_input || !hidden || !cell)) {
        set_error("%s: offsets, audio_input, hidden and cell must be non-null", where);
        return FA_INVALID_ARGUMENT;
    }
    if (count == 0) return FA_OK;
    if (offsets[0] < 0) {
        set_error("%s: offsets[0] is negative (%lld)", where, (long long)offsets[0]);
        return FA_INVALID_ARGUMENT;
    }
    for (int i = 0; i < count; ++i)
        if (offsets[i + 1] < offsets[i] || offsets[i + 1] > (1LL << 62)) {
            set_error("%s: offsets decrease at %d or pass 2^62 (%lld, %lld)", where, i, (long long)offsets[i],
                      (long long)offsets[i + 1]);
            return FA_INVALID_ARGUMENT;
        }
    const long long total_new = offsets[count] - offsets[0];
    if (total_new > 0 && !audio) {
        set_error("%s: audio is null with %lld samples", where, total_new);
        return FA_INVALID_ARGUMENT;
    }
    st = desc.reserve(std::max<size_t>((size_t)count * sizeof(InputJob), 4096));
    if (st != FA_OK) return st;
    HostStaging H(!device, stream);
    const float *src = nullptr;
    float *k_in, *k_h, *k_c;
    st = H.carve(d_io, [&](HostStaging::Layout &l) {
        src = l.in(total_new > 0 ? audio + offsets[0] : nullptr, (size_t)total_new);
        k_in = l.out(audio_input, (size_t)count * kModelInput);
        k_h = l.out(hidden, (size_t)count * kState);
        k_c = l.out(cell, (size_t)count * kState);
    });
    if (st != FA_OK) return st;
    InputJob *hj = static_cast<InputJob *>(desc.host.data());
    for (int i = 0; i < count; ++i) hj[i] = InputJob{offsets[i] - offsets[0], offsets[i + 1] - offsets[i], sessions[i]};
    st = desc.upload((size_t)count * sizeof(InputJob), stream);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(vad_model_inputs_kernel, count, kThreads, 0, stream,
                       static_cast<const InputJob *>(desc.device.data()), src, d_state.data(), d_meta.data(), k_in,
                       k_h, k_c));
    FA_CUDA_TRY(H.finish());
    for (int i = 0; i < count; ++i) table[sessions[i]].pending = true;
    return FA_OK;
}

int StreamSet::advance(int count, const int *sessions, const float *probability, const float *new_hidden,
                       const float *new_cell, const Resolved &r, bool device, int64_t *events) {
    const char *where = "fa_vad_stream_advance";
    int st = check_sessions(table, count, sessions, where);
    if (st != FA_OK) return st;
    if (count > 0 && (!probability || !new_hidden || !new_cell || !events)) {
        set_error("%s: probability, new_hidden, new_cell and events must be non-null", where);
        return FA_INVALID_ARGUMENT;
    }
    for (int i = 0; i < count; ++i)
        if (!table[sessions[i]].pending) {
            set_error("%s: session %d has no staged chunk", where, sessions[i]);
            return FA_INVALID_ARGUMENT;
        }
    if (count == 0) return FA_OK;
    st = desc.reserve(std::max<size_t>((size_t)count * sizeof(int), 4096));
    if (st != FA_OK) return st;
    HostStaging H(!device, stream);
    const float *k_p, *k_h, *k_c;
    long long *k_ev;
    st = H.carve(d_io, [&](HostStaging::Layout &l) {
        k_p = l.in(probability, (size_t)count);
        k_h = l.in(new_hidden, (size_t)count * kState);
        k_c = l.in(new_cell, (size_t)count * kState);
        k_ev = reinterpret_cast<long long *>(l.out(events, (size_t)count * 2));
    });
    if (st != FA_OK) return st;
    std::memcpy(desc.host.data(), sessions, (size_t)count * sizeof(int));
    st = desc.upload((size_t)count * sizeof(int), stream);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(vad_advance_kernel, count, kState, 0, stream, static_cast<const int *>(desc.device.data()), k_p,
                       k_h, k_c, d_state.data(), d_meta.data(), k_ev, r));
    FA_CUDA_TRY(H.finish());
    for (int i = 0; i < count; ++i) table[sessions[i]].pending = false;
    return FA_OK;
}

int StreamSet::state(int session, SessionInfo *info, float *context, float *hidden, float *cell) {
    int st = table.check(1, &session, "fa_vad_stream_session_state");
    if (st != FA_OK) return st;
    const float *S = d_state.data() + (size_t)session * kSlotFloats;
    long long m[kSlotFields];
    if (context) FA_CUDA_TRY(cudaMemcpyAsync(context, S, kContext * sizeof(float), cudaMemcpyDeviceToHost, stream));
    if (hidden)
        FA_CUDA_TRY(cudaMemcpyAsync(hidden, S + kHiddenAt, kState * sizeof(float), cudaMemcpyDeviceToHost, stream));
    if (cell) FA_CUDA_TRY(cudaMemcpyAsync(cell, S + kCellAt, kState * sizeof(float), cudaMemcpyDeviceToHost, stream));
    FA_CUDA_TRY(cudaMemcpyAsync(m, d_meta.data() + (size_t)session * kSlotFields, sizeof(m), cudaMemcpyDeviceToHost,
                                stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    *info = SessionInfo{m[kProcessed], m[kTempEnd], (int)m[kTriggered], table[session].pending ? 1 : 0};
    return FA_OK;
}

// ------------------------------------------------------------------------------------------------ clips
int clip_call(CallContext &C, bool fsmn, bool on_device, const float *input, const int64_t *offsets, int clips,
              const int64_t *total_samples, const Resolved &r, int64_t *counts, int64_t *segments, long long capacity,
              int64_t *total) {
    const char *entry = fsmn ? "fa_fsmn_vad_decide" : "fa_vad_segment";
    *total = 0;
    if (clips == 0) return FA_OK;
    const long long rows = offsets[clips];
    // descriptors, then room for the output offsets uploaded after the synchronisation
    std::vector<ClipDesc> cd((size_t)clips);
    long long pairs = 0;
    for (int b = 0; b < clips; ++b) {
        const long long n = offsets[b + 1] - offsets[b];
        cd[(size_t)b] = ClipDesc{offsets[b], n, pairs, fsmn ? 0 : total_samples[b]};
        pairs += fsmn ? fsmn_bound(n) : n;
    }
    const size_t desc_bytes = cd.size() * sizeof(ClipDesc);
    const size_t out_at = (desc_bytes + 255) & ~size_t(255);
    int st = C.stage.reserve(out_at + (size_t)clips * sizeof(long long));
    if (st != FA_OK) return st;
    std::memcpy(C.stage.host.data(), cd.data(), desc_bytes);
    st = C.stage.upload(desc_bytes, C.stream);
    if (st != FA_OK) return st;
    long long *d_scratch, *d_counts;
    st = carve_arena(C.scratch, [&](Carver &c) {
        d_scratch = c.take<long long>((size_t)std::max(1LL, 2 * pairs));
        d_counts = c.take<long long>((size_t)clips);
    });
    if (st != FA_OK) return st;
    st = C.h_buf.grow((size_t)clips * sizeof(long long));
    if (st != FA_OK) return st;
    HostStaging H(!on_device, C.stream);
    const float *d_in;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) { d_in = l.in(input, (size_t)rows); });
    if (st != FA_OK) return st;
    const char *d_desc = static_cast<const char *>(C.stage.device.data());
    const auto *d_clips = reinterpret_cast<const ClipDesc *>(d_desc);
    FA_CUDA_TRY(launch(vad_clip_kernel, dim3((unsigned)((clips + 127) / 128)), dim3(128), 0, C.stream, d_clips, clips,
                       d_in, fsmn ? 1 : 0, r, d_scratch, d_counts));
    auto *h_counts = static_cast<long long *>(C.h_buf.data());
    FA_CUDA_TRY(cudaMemcpyAsync(h_counts, d_counts, (size_t)clips * sizeof(long long), cudaMemcpyDeviceToHost,
                                C.stream));
    FA_CUDA_TRY(cudaStreamSynchronize(C.stream));
    long long *h_out_at = reinterpret_cast<long long *>(static_cast<char *>(C.stage.host.data()) + out_at);
    long long sum = 0;
    for (int b = 0; b < clips; ++b) {
        h_out_at[b] = sum;
        counts[b] = h_counts[b];
        sum += h_counts[b];
    }
    *total = sum;
    if (sum > capacity) {
        set_error("%s: %lld segments, capacity %lld", entry, sum, capacity);
        return FA_OUTPUT_TOO_SMALL;
    }
    if (sum == 0) return FA_OK;
    FA_CUDA_TRY(cudaMemcpyAsync(const_cast<char *>(d_desc) + out_at, h_out_at, (size_t)clips * sizeof(long long),
                                cudaMemcpyHostToDevice, C.stream));
    FA_CUDA_TRY(cudaEventRecord(C.stage.uploaded, C.stream));
    C.stage.in_flight = true;   // the next reserve() waits for this copy out of the pinned buffer
    HostStaging O(!on_device, C.stream);
    long long *d_out;
    st = O.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_out = reinterpret_cast<long long *>(l.out(segments, (size_t)(2 * sum)));
    });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(vad_gather_kernel, dim3((unsigned)clips), dim3(kThreads), 0, C.stream, d_clips, d_counts,
                       reinterpret_cast<const long long *>(d_desc + out_at), d_scratch, d_out));
    FA_CUDA_TRY(O.finish());
    return FA_OK;
}

} // namespace vad
} // namespace fa
