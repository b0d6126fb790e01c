// Placement of one centroid-linkage problem on the GPU, and the lane rule of the batch entry points: pure host
// functions of the problem's shape and the SM count, so that a CPU test can check every boundary (tests/emul).
//
// With max_workers worker CTAs (SMs - 1 for a single call), on a 132-SM H100 (W = 131):
//   master state in shared memory   level 3 (heap + nn + node_of) N <= 11 376, level 2 (heap + nn) <= 14 176,
//                                   level 1 (heap, uint16 indices) <= 18 808, level 0 (global, int heap) above
//   worker placement                resident when cap(D) * W >= N, cap(D) = node vectors per CTA (128 for D <= 219,
//                                   109 at D = 256, 11 at 2 048, 1 at 7 196); streamed from HBM otherwise, in
//                                   ceil(Ns / (W * 128)) <= 16 rounds per thread
//   limits (FA_RUNTIME_ERROR)       D >= 7 197 (cap(D) = 0: one target vector no longer fits) and
//                                   N > W * 2 048 (N rounded up to 32 exceeds W * 128 * 16 slots)
//   float32 filter                  N >= 2 048; pass 2 is the rows kernel when the per-tile bounds are kept
//                                   (N * ceil(N / 64) <= 2^24) and D <= 1 536, else the dense kernel
#pragma once

#include "fa_common.cuh"
#include <algorithm>

namespace fa {
namespace ahc {

constexpr int kMergeThreads = 128;   // scan threads per worker CTA: one slot each per round
constexpr int kMaxRounds = 16;       // streamed mode only: slots per thread

// Dynamic shared memory the merge kernel may use: leaves room for its static shared memory.
constexpr size_t kMergeSmemCap = 227 * 1024 - 2048;

// bytes of master state staged in shared memory at each level (must mirror ahc_master's carving)
inline size_t master_smem_bytes(int N, int level) {
    auto up = [](size_t b) { return (b + 15) & ~size_t(15); };
    const size_t words = (size_t)(2 * N - 1 + 31) >> 5;
    size_t b = up(sizeof(double) * N) + 2 * up(sizeof(uint16_t) * N) + up(sizeof(unsigned) * words);
    if (level >= 2) b += up(sizeof(int) * N);
    if (level >= 3) b += up(sizeof(int) * N);
    return b;
}

// Shared memory of one worker CTA before any resident node vector: the target vector and the reduction scratch.
inline size_t worker_fixed_smem(int D) {
    return 3 * sizeof(double) * (size_t)((D + 1) & ~1) + 2 * sizeof(double) * (kMergeThreads / 32) + 64;
}

// Node vectors one worker CTA can keep in shared memory (at most one per thread), 0 if not even one fits.
inline int resident_slot_capacity(int D) {
    const size_t fixed = worker_fixed_smem(D);
    if (fixed + sizeof(double) * D > kMergeSmemCap) return 0;
    return (int)std::min<size_t>(kMergeThreads, (kMergeSmemCap - fixed) / (sizeof(double) * (size_t)D));
}

// Test hooks (FA_AHC_* environment variables, read once per process in ahc_kernels.cu): fall-back placements and
// the float32 filter at small N.
struct Hooks {
    bool force_global = false, force_stream = false;
    int filter_min_n = 2048;   // problems at least this large take the float32 filter (0 = never)
};

struct Placement {
    int status = FA_OK;         // FA_OK, or FA_RUNTIME_ERROR: D too large (cap_slots == 0) or N above `capacity`
    int level = 0;              // master state in shared memory: 0 none, 1 heap, 2 + nn, 3 + node_of
    bool idx16 = false;         // heap indices are uint16_t (level >= 1)
    int cap_slots = 0;          // node vectors one worker CTA can keep in shared memory
    bool resident = false;      // every node vector in shared memory, else streamed from the k-major copy
    int workers = 0;            // worker CTAs (grid = workers + 1)
    int slots_per_cta = 0;      // resident only
    int rounds = 0;             // slots per scan thread
    long long capacity = 0;     // streamed only: slots the workers can scan, workers * 128 * 16
    size_t smem = 0;            // dynamic shared memory of the merge kernel
    bool filter = false;        // float32 filter of the initial nearest-neighbour pass
    bool keep_tmin = false;     // the filter keeps its per-tile bounds (N * ceil(N / 64) floats <= 64 MB)
    bool filter_rows = false;   // filter pass 2 is the rows kernel (else the dense kernel)
};

// Placement of an N x D problem (N >= 2) on at most max_workers worker CTAs.
inline Placement plan_linkage(int N, int D, int max_workers, const Hooks &hk) {
    Placement p;
    const int Ns = (N + 31) & ~31;
    // master placement: slot-indexed heap (+ nn, + node_of) in shared memory when it fits
    if (N <= 65535)
        for (int l = 1; l <= 3; ++l)
            if (master_smem_bytes(N, l) <= kMergeSmemCap) p.level = l;
    if (hk.force_global) p.level = 0;
    p.idx16 = p.level >= 1;
    // float32 filter of the initial nearest-neighbour pass
    p.filter = hk.filter_min_n > 0 && N >= hk.filter_min_n;
    const long long nt = (N + 63) / 64;
    p.keep_tmin = (long long)N * nt <= (16LL << 20);   // <= 64 MB
    p.filter_rows = p.keep_tmin && (size_t)8 * D * sizeof(float) <= 48 * 1024;
    // worker placement: resident (each CTA keeps <= 128 node vectors in shared memory) when the whole problem fits
    // into max_workers CTAs, else streamed from the k-major global copy
    p.cap_slots = resident_slot_capacity(D);
    if (p.cap_slots == 0) {
        p.status = FA_RUNTIME_ERROR;
        return p;
    }
    p.resident = (long long)p.cap_slots * max_workers >= N && !hk.force_stream;
    size_t worker_smem = worker_fixed_smem(D);
    if (p.resident) {
        // enough CTAs to hold every node, but no more than needed: the per-step barrier cost grows with CTA count
        p.workers = std::min(max_workers, std::max(1, (N + p.cap_slots - 1) / p.cap_slots));
        p.slots_per_cta = (N + p.workers - 1) / p.workers;
        p.rounds = 1;
        worker_smem += sizeof(double) * (size_t)D * p.slots_per_cta;
    } else {
        p.workers = std::max(1, std::min(max_workers, (Ns + kMergeThreads - 1) / kMergeThreads));
        p.rounds = (Ns + p.workers * kMergeThreads - 1) / (p.workers * kMergeThreads);
        p.capacity = (long long)p.workers * kMergeThreads * kMaxRounds;
        if (p.capacity < Ns) {
            p.status = FA_RUNTIME_ERROR;
            return p;
        }
    }
    p.smem = std::max(worker_smem, p.level ? master_smem_bytes(N, p.level) : (size_t)0);
    return p;
}

// Worker CTAs a problem needs to keep every node vector in shared memory (the fast placement), or 0 if a single CTA
// cannot hold even one vector.
inline int resident_workers_needed(int N, int D) {
    const int cap_slots = resident_slot_capacity(D);
    return cap_slots ? (N + cap_slots - 1) / cap_slots : 0;
}

// Batch of independent sets: `lanes` host threads run sets side by side, each on a solver capped at `worker_limit`
// worker CTAs (0: no cap, the single call's SMs - 1).
struct BatchLanes {
    int lanes = 1;
    int worker_limit = 0;
};

// As many sets at a time as still leaves each of them enough SMs to keep its node vectors in shared memory (the
// merge loop is ~3x slower when they are streamed from L2): 5 000 x 256 needs 46 workers + 1 master, so two sets run
// side by side on an H100's 132 SMs; small sets run four at a time.  A set too large to be resident even on the whole
// GPU is streamed, and the lane count then also keeps it within its lane's streamed capacity (worker_limit * 2 048
// slots); when no lane count above one does, the batch runs in one lane, exactly as one call per set would.
inline BatchLanes plan_batch_lanes(int set_count, long long n_max, int D, int sms) {
    BatchLanes b;
    b.lanes = std::max(1, std::min(set_count, 4));
    const int need = resident_workers_needed((int)std::min<long long>(n_max, 0x7fffffff), D);
    if (need > 0 && need + 1 <= sms) b.lanes = std::max(1, std::min(b.lanes, sms / (need + 1)));
    const long long ns_max = (n_max + 31) & ~31LL;
    for (; b.lanes > 1; --b.lanes) {
        const int limit = std::max(1, sms / b.lanes - 1);
        if ((long long)limit * kMergeThreads * kMaxRounds >= ns_max) break;
    }
    b.worker_limit = b.lanes == 1 ? 0 : std::max(1, sms / b.lanes - 1);
    return b;
}

} // namespace ahc
} // namespace fa
