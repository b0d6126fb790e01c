// The call context of every entry point that takes no handle (call_context.cu): clustering, the prepare stage, the
// resampler and per-feature normalisation each lease one per call from a pool and run on its stream and workspace.
#pragma once

#include "ahc_plan.h"
#include <functional>

namespace fa {

// One per concurrent caller, leased from a pool (the reference boundary is synchronous, stateless and re-entrant:
// FastClusterWrapper.cpp keeps no state, SURVEY §8b).  Buffers only grow: a context keeps the largest workspace any
// call on it has needed.
struct CallContext {
    int device = 0;
    Stream stream;   // declared first, so destroyed last: after every buffer
    ahc::Solver solver;
    UploadStage<> stage;        // launch descriptors of the prepare stage
    DeviceBuffer<> scratch;     // the prepare stage's counters, entry metadata and masks
    DeviceBuffer<> vbx_pool;    // scratch of VBx refinement, centroids and K-Means
    DeviceBuffer<> cent_pool;   // the pipeline's gamma / pi / ELBOs / centroids
    DeviceBuffer<> d_buf;       // inputs and outputs of one call
    PinnedBuffer<> h_buf;
    Event ev[6];   // pipeline timing: before normalisation, before / after AHC, before VBx, before centroids, after assignment
    bool ready = false;
    int worker_limit = 0;

    // on the current device: stream, events, solver and the clustering kernels' shared-memory maxima
    int init(int worker_limit);
};

// Leases a context of the current device for `worker_limit` (from the pool, or made), runs body on it and returns the
// body's status.  A context whose call ended in FA_CUDA_ERROR is freed rather than pooled.
int with_context(int worker_limit, const std::function<int(CallContext &)> &body);

} // namespace fa
