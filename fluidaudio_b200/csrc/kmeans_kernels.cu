// K-Means re-clustering to a forced speaker count (SURVEY.md 8f rank 4), device-resident.
//
// Reference: KMeansClustering.clusterWithCentroids / clusterWithCentroidsNInit
// (Sources/FluidAudio/Diarizer/Offline/Clustering/KMeansClustering.swift:39-130), SeededRNG (:212-223),
// used by VBxClustering.refineWithConstraints (VBxClustering.swift:685-733) when SpeakerCountConstraints bind.
// The Swift standard library's shuffle / randomElement / next(upperBound:) (Lemire's method) are restated here the
// way DESIGN.md section 2 documents them (a third-party dependency of the reference, not vendored in it).
//
// Arithmetic order = the oracle's: every squared distance and every norm is one thread's sequential sum with
// individually rounded operations; centroid sums run over the points in index order (one thread per (cluster, dim)).
// All iterations of a run are enqueued without a host round trip: a device-side `done` flag turns the remaining
// launches into no-ops once the assignment repeats (the reference's `break`), and the host looks at the flag every
// few iterations only to stop enqueuing.  The single-threaded parts (seeded shuffle, re-seeding of empty clusters,
// the inertia sum) are what the reference defines sequentially.
#include "kmeans_plan.h"

#include <algorithm>
#include <cfloat>
#include <climits>
#include <cstdint>
#include <vector>

namespace fa {
namespace kmeans {

struct Lcg {
    unsigned long long state;
    __host__ __device__ unsigned long long next() {
        state = state * 6364136223846793005ull + 1442695040888963407ull;
        return state;
    }
    __device__ unsigned long long next_below(unsigned long long upper) {   // Lemire, as Swift's next(upperBound:)
        unsigned long long r = next();
        unsigned long long hi = __umul64hi(r, upper), lo = r * upper;
        if (lo < upper) {
            const unsigned long long t = (0ull - upper) % upper;
            while (lo < t) {
                r = next();
                hi = __umul64hi(r, upper);
                lo = r * upper;
            }
        }
        return hi;
    }
};

struct RunState {
    unsigned long long rng;
    int done;        // assignment repeated: everything after is a no-op
    int changed;     // set by the assignment kernel of the current iteration
    int iterations;
    double inertia;
};

// normalizeEmbeddings (:133-145): x / ||x|| when ||x|| > 1e-10, else unchanged
__global__ void normalize_kernel(const double *__restrict__ emb, int N, int D, double *__restrict__ x) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const double *r = emb + (size_t)i * D;
    double s = 0.0;
    for (int k = 0; k < D; ++k) s = __dadd_rn(s, __dmul_rn(r[k], r[k]));
    const double norm = __dsqrt_rn(s);
    double *o = x + (size_t)i * D;
    if (norm > 1e-10) {
        const double inv = __ddiv_rn(1.0, norm);
        for (int k = 0; k < D; ++k) o[k] = __dmul_rn(r[k], inv);
    } else {
        for (int k = 0; k < D; ++k) o[k] = r[k];
    }
}

// k-major copy for coalesced thread-per-point scans
__global__ void transpose_kernel(const double *__restrict__ x, int N, int D, double *__restrict__ xt) {
    __shared__ double tile[32][33];
    const int i0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int i = i0 + r, k = k0 + threadIdx.x;
        tile[r][threadIdx.x] = (i < N && k < D) ? x[(size_t)i * D + k] : 0.0;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int k = k0 + r, i = i0 + threadIdx.x;
        if (i < N && k < D) xt[(size_t)k * N + i] = tile[threadIdx.x][r];
    }
}

// start of a run: centroids = the first k entries of the seeded shuffle (done on the host, initializeCentroids
// :147-155), previous assignment = all zeros (:68), fresh run state carrying the generator's state after the shuffle
__global__ void init_run_kernel(const double *__restrict__ x, int N, int D, int k, const int *__restrict__ picks,
                                unsigned long long rng_state, double *cent, int *labels_prev, RunState *st) {
    if (threadIdx.x == 0) {
        st->rng = rng_state;
        st->done = 0;
        st->changed = 0;
        st->iterations = 0;
        st->inertia = 0.0;
    }
    for (int j = 0; j < k; ++j)
        for (int q = threadIdx.x; q < D; q += blockDim.x) cent[(size_t)j * D + q] = x[(size_t)picks[j] * D + q];
    for (int i = threadIdx.x; i < N; i += blockDim.x) labels_prev[i] = 0;
}

// assignToCentroids (:161-176) + comparison with the previous assignment
__global__ void assign_kernel(const double *__restrict__ xt, int N, int D, const double *__restrict__ cent, int k,
                              const int *__restrict__ prev, int *__restrict__ fresh, RunState *st) {
    if (st->done) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    int best = 0;
    double bd = DBL_MAX;
    for (int j = 0; j < k; ++j) {
        const double *c = cent + (size_t)j * D;
        double s = 0.0;
        for (int q = 0; q < D; ++q) {
            const double t = __dsub_rn(xt[(size_t)q * N + i], __ldg(c + q));
            s = __dadd_rn(s, __dmul_rn(t, t));
        }
        if (s < bd) {
            bd = s;
            best = j;
        }
    }
    fresh[i] = best;
    if (best != prev[i]) st->changed = 1;
}

// updateCentroids (:187-210) for clusters that kept members; one thread per (cluster, dimension)
__global__ void update_kernel(const double *__restrict__ x, int N, int D, const int *__restrict__ labels, int k,
                              double *cent, int *counts, const RunState *st) {
    if (st->done || !st->changed) return;
    const int j = blockIdx.y, q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= D) return;
    double s = 0.0;
    int cnt = 0;
    for (int i = 0; i < N; ++i)
        if (labels[i] == j) {
            s = __dadd_rn(s, x[(size_t)i * D + q]);
            ++cnt;
        }
    if (q == 0) counts[j] = cnt;
    if (cnt > 0) cent[(size_t)j * D + q] = __dmul_rn(s, __ddiv_rn(1.0, (double)cnt));
}

// end of an iteration: the reference's `break`, or re-seeding of empty clusters in cluster order, then bookkeeping
__global__ void finish_iteration_kernel(const double *__restrict__ x, int N, int D, int k, double *cent,
                                        const int *counts, RunState *st) {
    __shared__ int pick[1024];
    __shared__ int stop;
    if (threadIdx.x == 0) {
        stop = 0;
        if (st->done) {
            stop = 1;
        } else if (!st->changed) {
            st->done = 1;                       // newAssignments == assignments: keep the centroids, leave the loop
            stop = 1;
        } else {
            Lcg g{st->rng};
            for (int j = 0; j < k; ++j) pick[j] = counts[j] > 0 ? -1 : (int)g.next_below((unsigned long long)N);
            st->rng = g.state;
            st->iterations += 1;
            st->changed = 0;
        }
    }
    __syncthreads();
    if (stop) return;
    for (int j = 0; j < k; ++j)
        if (pick[j] >= 0)
            for (int q = threadIdx.x; q < D; q += blockDim.x) cent[(size_t)j * D + q] = x[(size_t)pick[j] * D + q];
}

// inertia = sum_i ||x_i - c_{label_i}||^2 (:118-121): distances in parallel, the sum in index order
__global__ void point_inertia_kernel(const double *__restrict__ xt, int N, int D, const double *__restrict__ cent, int k,
                                     const int *__restrict__ labels, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int j = labels[i];
    double s = 0.0;
    if (j >= 0 && j < k) {
        const double *c = cent + (size_t)j * D;
        for (int q = 0; q < D; ++q) {
            const double t = __dsub_rn(xt[(size_t)q * N + i], __ldg(c + q));
            s = __dadd_rn(s, __dmul_rn(t, t));
        }
    }
    out[i] = s;
}
__global__ void sum_inertia_kernel(const double *__restrict__ per_point, int N, RunState *st) {
    double s = 0.0;
    for (int i = 0; i < N; ++i) s = __dadd_rn(s, per_point[i]);
    st->inertia = s;
}
__global__ void iota_kernel(int *labels, int N) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) labels[i] = i;
}

namespace {
// host twin of Lcg::next_below (Swift's next(upperBound:), Lemire's method on the 128-bit product)
unsigned long long host_next_below(Lcg &g, unsigned long long upper) {
    unsigned __int128 m = (unsigned __int128)g.next() * upper;
    if ((unsigned long long)m < upper) {
        const unsigned long long t = (0ull - upper) % upper;
        while ((unsigned long long)m < t) m = (unsigned __int128)g.next() * upper;
    }
    return (unsigned long long)(m >> 64);
}
} // namespace

void resolve_constraints(long long num_embeddings, long long num_speakers, long long min_speakers, long long max_speakers,
                         long long *lo_out, long long *hi_out) {
    // SpeakerCountConstraints.resolve (SpeakerCountConstraints.swift:27-71)
    auto has = [](long long v) { return v != (long long)INT32_MIN; };   // FA_NO_VALUE
    long long lo = has(num_speakers) ? num_speakers : (has(min_speakers) ? min_speakers : 1);
    lo = std::max(1LL, std::min(num_embeddings, lo));
    long long hi = has(num_speakers) ? num_speakers : (has(max_speakers) ? max_speakers : num_embeddings);
    hi = std::max(1LL, std::min(num_embeddings, hi));
    if (lo > hi) lo = hi;
    *lo_out = lo;
    *hi_out = hi;
}

int cluster_ninit_device(vbx::Workspace &ws, const double *d_emb, int N, int D, int num_clusters, int max_iterations,
                         int n_init, unsigned long long base_seed, int *d_labels, double *d_centroids, int *rows,
                         int *best_init, cudaStream_t s, long long *launches) {
    long long lc = 0;
    if (rows) *rows = 0;
    if (best_init) *best_init = 0;
    if (N <= 0) return FA_OK;
    if (D <= 0) {
        FA_CUDA_TRY(cudaMemsetAsync(d_labels, 0, sizeof(int) * N, s));
        return FA_OK;
    }
    const int k = std::min(num_clusters, N);
    if (k <= 0) {
        FA_CUDA_TRY(cudaMemsetAsync(d_labels, 0, sizeof(int) * N, s));
        return FA_OK;
    }
    if (N <= k) {                                             // :60-62: identity, centroids = the raw embeddings
        iota_kernel<<<(N + 255) / 256, 256, 0, s>>>(d_labels, N);
        FA_CUDA_TRY(cudaGetLastError());
        FA_CUDA_TRY(cudaMemcpyAsync(d_centroids, d_emb, sizeof(double) * (size_t)N * D, cudaMemcpyDeviceToDevice, s));
        if (rows) *rows = N;
        if (launches) *launches += 1;
        return FA_OK;
    }
    if (k > 1024) {
        fa::set_error("K-Means re-clustering supports at most 1024 clusters, got %d", k);
        return FA_UNSUPPORTED;
    }
    const int runs = (N > num_clusters && n_init > 1) ? n_init : 1;   // :106-110
    size_t need;
    {
        Carver c{nullptr};
        c.take<double>((size_t)N * D);
        c.take<double>((size_t)N * D);
        c.take<double>((size_t)k * D);
        c.take<double>((size_t)N);
        c.take<int>((size_t)N * 3);
        c.take<int>((size_t)k);
        c.take<RunState>(1);
        need = c.off + 4096;
    }
    int st = ws.reserve(std::max(ws.pool_bytes, need));
    if (st != FA_OK) return st;
    Carver c{static_cast<char *>(ws.pool)};
    double *d_x = c.take<double>((size_t)N * D);
    double *d_xt = c.take<double>((size_t)N * D);
    double *d_cent = c.take<double>((size_t)k * D);
    double *d_pp = c.take<double>((size_t)N);
    int *d_perm = c.take<int>(N);
    int *d_lab[2] = {c.take<int>(N), c.take<int>(N)};
    int *d_counts = c.take<int>(k);
    RunState *d_state = c.take<RunState>(1);

    normalize_kernel<<<(N + 127) / 128, 128, 0, s>>>(d_emb, N, D, d_x);
    FA_CUDA_TRY(cudaGetLastError());
    transpose_kernel<<<dim3((N + 31) / 32, (D + 31) / 32), dim3(32, 8), 0, s>>>(d_x, N, D, d_xt);
    FA_CUDA_TRY(cudaGetLastError());
    lc += 2;

    double best = DBL_MAX;
    RunState h{};
    std::vector<int> perm(N);
    for (int run = 0; run < runs; ++run) {
        // indices.shuffle(using: &rng) — O(N) integer work on the host, like the heapify of the AHC path
        Lcg g{base_seed + (unsigned long long)run};
        for (int i = 0; i < N; ++i) perm[i] = i;
        for (int amount = N, cur = 0; amount > 1; ++cur) {
            const int r = (int)host_next_below(g, (unsigned long long)amount);
            amount -= 1;
            std::swap(perm[cur], perm[cur + r]);
        }
        FA_CUDA_TRY(cudaMemcpyAsync(d_perm, perm.data(), sizeof(int) * k, cudaMemcpyHostToDevice, s));
        FA_CUDA_TRY(cudaStreamSynchronize(s));   // perm is reused by the next run
        init_run_kernel<<<1, 256, 0, s>>>(d_x, N, D, k, d_perm, g.state, d_cent, d_lab[1], d_state);
        FA_CUDA_TRY(cudaGetLastError());
        lc += 1;
        int it = 0;
        bool done = false;
        while (it < max_iterations && !done) {
            const int batch = std::min(8, max_iterations - it);
            for (int b = 0; b < batch; ++b, ++it) {
                int *fresh = d_lab[it & 1], *prev = d_lab[(it & 1) ^ 1];
                assign_kernel<<<(N + 127) / 128, 128, 0, s>>>(d_xt, N, D, d_cent, k, prev, fresh, d_state);
                update_kernel<<<dim3((D + 127) / 128, k), 128, 0, s>>>(d_x, N, D, fresh, k, d_cent, d_counts, d_state);
                finish_iteration_kernel<<<1, 256, 0, s>>>(d_x, N, D, k, d_cent, d_counts, d_state);
                lc += 3;
            }
            FA_CUDA_TRY(cudaGetLastError());
            FA_CUDA_TRY(cudaMemcpyAsync(&h, d_state, sizeof(RunState), cudaMemcpyDeviceToHost, s));
            FA_CUDA_TRY(cudaStreamSynchronize(s));
            done = h.done != 0;
        }
        // the assignment the reference returns: the last one computed.  With the `break` that is the buffer written
        // in iteration `iterations` (equal to the previous one); after max_iterations full rounds it is the last.
        const int last = h.done ? h.iterations : (max_iterations - 1);
        const int *final_labels = max_iterations > 0 ? d_lab[last & 1] : d_lab[1];
        point_inertia_kernel<<<(N + 127) / 128, 128, 0, s>>>(d_xt, N, D, d_cent, k, final_labels, d_pp);
        sum_inertia_kernel<<<1, 1, 0, s>>>(d_pp, N, d_state);
        lc += 2;
        FA_CUDA_TRY(cudaGetLastError());
        FA_CUDA_TRY(cudaMemcpyAsync(&h, d_state, sizeof(RunState), cudaMemcpyDeviceToHost, s));
        FA_CUDA_TRY(cudaStreamSynchronize(s));
        // :122-125: strictly lower inertia wins.  Run 0 (the base seed) is always taken first, so a NaN inertia in every
        // run (a NaN row makes every distance NaN) returns the base-seed run; a later run beats it only by comparing
        // below `best`, which a NaN inertia never lowers.
        const bool better = h.inertia < best;
        if (run == 0 || better) {
            if (better) best = h.inertia;
            FA_CUDA_TRY(cudaMemcpyAsync(d_labels, final_labels, sizeof(int) * N, cudaMemcpyDeviceToDevice, s));
            FA_CUDA_TRY(cudaMemcpyAsync(d_centroids, d_cent, sizeof(double) * (size_t)k * D, cudaMemcpyDeviceToDevice, s));
            if (best_init) *best_init = run;
        }
    }
    FA_CUDA_TRY(cudaStreamSynchronize(s));
    if (rows) *rows = k;
    if (launches) *launches += lc;
    return FA_OK;
}

} // namespace kmeans
} // namespace fa
