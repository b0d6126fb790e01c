// Diarizer timelines (fa_diarizer_timeline_*): DiarizerTimeline's numeric core (DiarizerTimeline.swift) for any number
// of sessions in HBM, each with its per-speaker SegmentScratch, a ring of its last maxStoredFrames finalized rows and its
// tentative rows.
//
// Every length follows from the row counts alone, never from values: the host mirrors each session's finalized cursor
// and tentative row count, and bounds the segments a push can emit (segment_bound, timeline_core.cuh).  A push therefore
// checks and plans every session before anything runs, uploads one descriptor per session and issues two launches
// (timeline_kernels.cu); the host variant stages its arrays in the set's one staging buffer (HostStaging,
// fa_common.cuh) and adds their copies and two synchronisations, one for the counts and one for exactly the segments.
// The scratches, which depend on values, stay on the device.
#include "timeline_plan.h"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace fa {
namespace timeline {

constexpr long long kMaxRowsPerPush = 1LL << 30;   // per session; keeps every lane's segment count in an int

int check_config(const Config &c, int max_tentative_rows) {
    if (c.num_speakers < 1 || c.num_speakers > kMaxSpeakers) {
        fa::set_error("diarizer timeline config: numSpeakers %d outside 1..%d", c.num_speakers, kMaxSpeakers);
        return FA_INVALID_ARGUMENT;
    }
    if (c.pad_on < 0 || c.pad_off < 0 || c.min_on < 0 || c.min_off < 0) {
        fa::set_error("diarizer timeline config: onset / offset pad frames and minFramesOn / Off must be >= 0");
        return FA_INVALID_ARGUMENT;
    }
    if (!std::isfinite(c.onset) || !std::isfinite(c.offset) || !std::isfinite(c.frame_duration)) {
        fa::set_error("diarizer timeline config: thresholds and frameDurationSeconds must be finite");
        return FA_INVALID_ARGUMENT;
    }
    if (c.activity != kSigmoids && c.activity != kLogits) {
        fa::set_error("diarizer timeline config: unknown activity type %d", c.activity);
        return FA_INVALID_ARGUMENT;
    }
    if (c.max_stored < 0 || max_tentative_rows < 0) {
        fa::set_error("diarizer timeline config: maxStoredFrames (%d) and max_tentative_rows (%d) must be >= 0",
                      c.max_stored, max_tentative_rows);
        return FA_INVALID_ARGUMENT;
    }
    return FA_OK;
}

int TimelineSet::init(const Config &c, int max_tentative_rows) {
    cfg = c;
    layout = Layout{c.num_speakers, c.max_stored, max_tentative_rows,
                    ((long long)c.max_stored + max_tentative_rows) * c.num_speakers};
    return stream.create();
}

int TimelineSet::open(int *session) {
    auto grow = [&](int grown) {
        return grow_slots(table.slots(), grown, stream, d_scratch, (size_t)layout.speakers, d_rows,
                          (size_t)layout.slot_floats);
    };
    // DiarizerTimeline.init: fresh scratches, no predictions, cursor 0 (the mirror's value-initialised state)
    auto init = [&](int id) -> int {
        FA_CUDA_TRY(cudaMemsetAsync(d_scratch.data() + (size_t)id * layout.speakers, 0,
                                    layout.speakers * sizeof(StoredScratch), stream));
        return FA_OK;
    };
    return table.open(16, grow, init, session);
}

int TimelineSet::close(int session) { return table.close(session, "diarizer timeline"); }

int TimelineSet::push(int count, const int *sessions, const float *fin, const int64_t *fin_rows, const float *ten,
                      const int64_t *ten_rows, bool on_device, Segment *fin_out, long long fin_cap, Segment *ten_out,
                      long long ten_cap, int64_t *fin_counts, int64_t *ten_counts) {
    if (count < 0 || (count > 0 && (!sessions || !fin_rows || !ten_rows || !fin_counts || !ten_counts))) {
        fa::set_error("diarizer timeline push: count must be >= 0; sessions, row counts and counts non-null");
        return FA_INVALID_ARGUMENT;
    }
    if (count == 0) return FA_OK;
    int st = table.check(count, sessions, "diarizer timeline push");
    if (st != FA_OK) return st;
    const int S = layout.speakers;
    std::vector<TimelineSession> next(count);
    long long nsum = 0, msum = 0, fin_bound = 0, ten_bound = 0, stage = 0;
    for (int i = 0; i < count; ++i) {
        const long long n = fin_rows[i], m = ten_rows[i];
        if (n < 0 || m < 0 || n > kMaxRowsPerPush || m > layout.tentative_rows) {
            fa::set_error("diarizer timeline push: session %d: %lld finalized rows (0..2^30) and %lld tentative rows "
                          "(0..max_tentative_rows = %lld)", sessions[i], n, m, layout.tentative_rows);
            return FA_INVALID_ARGUMENT;
        }
        next[i] = TimelineSession{table[sessions[i]].cursor + n, m};
        nsum += n;
        msum += m;
        fin_bound += S * finalized_bound(n);
        ten_bound += S * tentative_bound(m);
        stage += S * segment_bound(n, m);
    }
    if ((nsum > 0 && !fin) || (msum > 0 && !ten)) {
        fa::set_error("diarizer timeline push: finalized / tentative rows are null");
        return FA_INVALID_ARGUMENT;
    }
    if ((fin_bound > 0 && (!fin_out || fin_cap < fin_bound)) || (ten_bound > 0 && (!ten_out || ten_cap < ten_bound))) {
        fa::set_error("diarizer timeline push: outputs need %lld finalized and %lld tentative segments, buffers hold %lld "
                      "and %lld", fin_bound, ten_bound, fin_out ? fin_cap : 0, ten_out ? ten_cap : 0);
        return FA_INVALID_ARGUMENT;
    }

    // ---- buffers and descriptors (the host variant's counts are one scratch array: one copy reads them all back)
    HostStaging H(!on_device, stream);
    const float *f, *t;
    Segment *f_out, *t_out;
    int64_t *d_counts = nullptr;
    const int lanes = count * S;
    const size_t desc_bytes = (size_t)count * sizeof(PushJob);
    st = push_desc.reserve(std::max<size_t>(desc_bytes, 4096));
    if (st == FA_OK) st = d_stage.grow((size_t)std::max(stage, 1LL) * sizeof(Segment));
    if (st == FA_OK) st = d_lane_counts.grow((size_t)2 * lanes * sizeof(int));
    if (st == FA_OK) st = d_lane_offsets.grow((size_t)2 * lanes * sizeof(long long));
    if (st == FA_OK)
        st = H.carve(staging, [&](HostStaging::Layout &l) {
            f = l.in(fin, (size_t)(nsum * S));
            t = l.in(ten, (size_t)(msum * S));
            f_out = l.out(fin_out, (size_t)fin_bound);
            t_out = l.out(ten_out, (size_t)ten_bound);
            if (!on_device) d_counts = l.take<int64_t>(2 * (size_t)count);
        });
    if (st != FA_OK) return st;
    PushJob *hj = static_cast<PushJob *>(push_desc.host.data());
    long long fo = 0, to = 0, so = 0;
    for (int i = 0; i < count; ++i) {
        const long long n = fin_rows[i], m = ten_rows[i], b = segment_bound(n, m);
        hj[i] = PushJob{sessions[i], table[sessions[i]].cursor, n, m, fo * S, to * S, so, b, (long long)i * S};
        fo += n;
        to += m;
        so += S * b;
    }

    // ---- device work, on the handle's stream
    int64_t *f_cnt = on_device ? fin_counts : d_counts, *t_cnt = on_device ? ten_counts : d_counts + count;
    st = push_desc.upload(desc_bytes, stream);
    if (st == FA_OK) {
        const PushJob *jobs = static_cast<const PushJob *>(push_desc.device.data());
        st = launch_push(cfg, layout, jobs, count, f, t, d_scratch.data(), d_rows.data(), d_stage.data(),
                         d_lane_counts.data(), f_cnt, t_cnt, stream);
        if (st == FA_OK)
            st = launch_pack(layout, lanes, jobs, d_stage.data(), d_lane_counts.data(), d_lane_offsets.data(), f_out, t_out,
                             stream);
    }
    if (st != FA_OK) return st;
    if (!on_device) {
        std::vector<int64_t> counts(2 * (size_t)count);
        FA_CUDA_TRY(cudaMemcpyAsync(counts.data(), f_cnt, counts.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, stream));
        FA_CUDA_TRY(cudaStreamSynchronize(stream));
        std::memcpy(fin_counts, counts.data(), (size_t)count * sizeof(int64_t));
        std::memcpy(ten_counts, counts.data() + count, (size_t)count * sizeof(int64_t));
        long long nf = 0, nt = 0;
        for (int i = 0; i < count; ++i) {
            nf += fin_counts[i];
            nt += ten_counts[i];
        }
        FA_CUDA_TRY(H.back(fin_out, f_out, (size_t)nf));
        FA_CUDA_TRY(H.back(ten_out, t_out, (size_t)nt));
        if (nf || nt) FA_CUDA_TRY(H.sync());
    }
    table.commit(count, sessions, next.data());
    return FA_OK;
}

int TimelineSet::finalize(int count, const int *sessions) {
    if (count < 0 || (count > 0 && !sessions)) {
        fa::set_error("diarizer timeline finalize: count must be >= 0 and sessions non-null");
        return FA_INVALID_ARGUMENT;
    }
    if (count == 0) return FA_OK;
    int st = table.check(count, sessions, "diarizer timeline finalize");
    if (st != FA_OK) return st;
    // _finalizeUnlocked (DiarizerTimeline.swift:883-891): the tentative rows join the stored ones, the cursor advances
    std::vector<TimelineSession> next(count);
    std::vector<FinalizeJob> jobs;
    for (int i = 0; i < count; ++i) {
        const TimelineSession &m = table[sessions[i]];
        next[i] = TimelineSession{m.cursor + m.tentative, 0};
        if (m.tentative > 0 && layout.ring_rows > 0) jobs.push_back(FinalizeJob{sessions[i], m.cursor, m.tentative});
    }
    if (!jobs.empty()) {
        const size_t bytes = jobs.size() * sizeof(FinalizeJob);
        st = finalize_desc.reserve(std::max<size_t>(bytes, 4096));
        if (st != FA_OK) return st;
        std::memcpy(finalize_desc.host.data(), jobs.data(), bytes);
        st = finalize_desc.upload(bytes, stream);
        if (st == FA_OK)
            st = launch_finalize(layout, static_cast<const FinalizeJob *>(finalize_desc.device.data()), (int)jobs.size(),
                                 d_rows.data(), stream);
        if (st != FA_OK) return st;
    }
    table.commit(count, sessions, next.data());
    return FA_OK;
}

int TimelineSet::reset(int count, const int *sessions) {
    if (count < 0 || (count > 0 && !sessions)) {
        fa::set_error("diarizer timeline reset: count must be >= 0 and sessions non-null");
        return FA_INVALID_ARGUMENT;
    }
    int st = table.check(count, sessions, "diarizer timeline reset");
    if (st != FA_OK) return st;
    // _resetUnlocked (:921-934): no predictions, cursor 0, fresh scratches
    for (int i = 0; i < count; ++i)
        FA_CUDA_TRY(cudaMemsetAsync(d_scratch.data() + (size_t)sessions[i] * layout.speakers, 0,
                                    layout.speakers * sizeof(StoredScratch), stream));
    std::vector<TimelineSession> next(count, TimelineSession{0, 0});
    table.commit(count, sessions, next.data());
    return FA_OK;
}

int TimelineSet::clear_speaker(int session, int speaker) {
    int st = table.check(1, &session, "diarizer timeline clear speaker");
    if (st != FA_OK) return st;
    if (speaker < 0 || speaker >= layout.speakers) {
        fa::set_error("diarizer timeline clear speaker: speaker %d outside 0..%d", speaker, layout.speakers - 1);
        return FA_INVALID_ARGUMENT;
    }
    // scratches[index] = SegmentScratch() (:1108-1111, :1134-1136)
    FA_CUDA_TRY(cudaMemsetAsync(d_scratch.data() + (size_t)session * layout.speakers + speaker, 0, sizeof(StoredScratch),
                                stream));
    return FA_OK;
}

int TimelineSet::state(int session, SessionInfo *info, float *stored, float *tentative, Scratch *scratch) {
    if (!table.valid(session) || !info) {
        fa::set_error("diarizer timeline state: session %d is not open (or info is null)", session);
        return FA_INVALID_ARGUMENT;
    }
    const TimelineSession &m = table[session];
    const int S = layout.speakers;
    const long long R = layout.ring_rows, fill = std::min(m.cursor, R);
    const float *rows = d_rows.data() + (size_t)session * layout.slot_floats;
    if (stored && fill) {
        // frames [cursor - fill, cursor) from ring row (cursor - fill) % R on, in two runs
        const long long head = (m.cursor - fill) % R, first = std::min(fill, R - head);
        FA_CUDA_TRY(cudaMemcpyAsync(stored, rows + head * S, first * S * sizeof(float), cudaMemcpyDeviceToHost, stream));
        if (fill > first)
            FA_CUDA_TRY(cudaMemcpyAsync(stored + first * S, rows, (fill - first) * S * sizeof(float),
                                        cudaMemcpyDeviceToHost, stream));
    }
    if (tentative && m.tentative)
        FA_CUDA_TRY(cudaMemcpyAsync(tentative, rows + R * S, m.tentative * S * sizeof(float), cudaMemcpyDeviceToHost,
                                    stream));
    std::vector<StoredScratch> sc(S);
    FA_CUDA_TRY(cudaMemcpyAsync(sc.data(), d_scratch.data() + (size_t)session * S, S * sizeof(StoredScratch),
                                cudaMemcpyDeviceToHost, stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    if (scratch)
        for (int k = 0; k < S; ++k) scratch[k] = load_scratch(sc[k]);
    *info = SessionInfo{m.cursor, fill, m.tentative};
    return FA_OK;
}

} // namespace timeline
} // namespace fa
