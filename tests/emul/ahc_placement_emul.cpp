// The merge kernel's placement and the batch lane rule (fluidaudio_b200/csrc/ahc_placement.h), compiled on the host for
// the CPU test-suite.
//   extern "C" void ahc_placement(int N, int D, int max_workers, int force_global, int force_stream, int filter_min_n,
//                                 long long out[13])
//       out = status, level, idx16, cap_slots, resident, workers, slots_per_cta, rounds, capacity, smem, filter,
//             keep_tmin, filter_rows
//   extern "C" void ahc_batch_lanes(int set_count, long long n_max, int D, int sms, int out[2])   -> lanes, worker_limit
#include "../../fluidaudio_b200/csrc/ahc_placement.h"

using namespace fa::ahc;

extern "C" void ahc_placement(int N, int D, int max_workers, int force_global, int force_stream, int filter_min_n,
                              long long *out) {
    Hooks hk;
    hk.force_global = force_global != 0;
    hk.force_stream = force_stream != 0;
    hk.filter_min_n = filter_min_n;
    const Placement p = plan_linkage(N, D, max_workers, hk);
    const long long v[13] = {p.status, p.level, p.idx16, p.cap_slots, p.resident, p.workers, p.slots_per_cta,
                             p.rounds, p.capacity, (long long)p.smem, p.filter, p.keep_tmin, p.filter_rows};
    for (int i = 0; i < 13; ++i) out[i] = v[i];
}

extern "C" void ahc_batch_lanes(int set_count, long long n_max, int D, int sms, int *out) {
    const BatchLanes b = plan_batch_lanes(set_count, n_max, D, sms);
    out[0] = b.lanes;
    out[1] = b.worker_limit;
}
