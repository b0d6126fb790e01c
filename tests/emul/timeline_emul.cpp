// Host run of the diarizer timelines' per-lane arithmetic (fluidaudio_b200/csrc/timeline_core.cuh; CPU test-suite
// only): one push of one session, each speaker through push_lane as a lane of timeline_scan_kernel runs it, its segments
// staged per lane and then packed speaker-major as timeline_pack_kernel packs them.
//   timeline_emul_push(ints {S, pad_on, pad_off, min_on, min_off, activity}, floats {onset, offset},
//                      scratch [S] in/out, cursor, fin [n x S], n, ten [m x S], m, fin_out, ten_out, counts[2],
//                      lane_total [S]: each lane's segment count, for the per-push bound)
#include "../../fluidaudio_b200/csrc/timeline_core.cuh"

#include <vector>

using namespace fa::timeline;

extern "C" void timeline_emul_push(const int *ints, const float *floats, Scratch *scratch, long long cursor,
                                   const float *fin, long long n, const float *ten, long long m, Segment *fin_out,
                                   Segment *ten_out, long long *counts, long long *lane_total) {
    const int S = ints[0];
    const Params c{floats[0], floats[1], ints[1], ints[2], ints[3], ints[4], ints[5]};
    std::vector<std::vector<Segment>> f(S), t(S);
    for (int k = 0; k < S; ++k) {
        auto emit = [&](const Segment &s, bool finalized) { (finalized ? f[k] : t[k]).push_back(s); };
        push_lane(c, scratch[k], k, cursor, n, [&](long long i) { return fin[i * S + k]; }, m,
                  [&](long long i) { return ten[i * S + k]; }, emit);
        lane_total[k] = (long long)(f[k].size() + t[k].size());
    }
    counts[0] = counts[1] = 0;
    for (int k = 0; k < S; ++k) {
        for (const Segment &s : f[k]) fin_out[counts[0]++] = s;
        for (const Segment &s : t[k]) ten_out[counts[1]++] = s;
    }
}
