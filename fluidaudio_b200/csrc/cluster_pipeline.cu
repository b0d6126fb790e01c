// Clustering host code: the diarization pipeline (OfflineDiarizerManager.cluster(_:) :286-375) in its
// steps, the batch lanes and the standalone stages.  The kernels are in ahc_kernels.cu, vbx_kernels.cu and kmeans_kernels.cu.
#include "cluster_plan.h"
#include "assign_host.h"
#include "kmeans_plan.h"
#include "vbx_plan.h"
#include "c_abi.h"

#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <thread>
#include <vector>

namespace fa {

static vbx::Config to_vbx(const fa_vbx_config &c) {
    vbx::Config vc;
    vc.Fa = c.Fa;
    vc.Fb = c.Fb;
    vc.max_iterations = c.max_iterations;
    vc.epsilon = c.epsilon;
    vc.init_smoothing = c.init_smoothing;
    return vc;
}

static float ms_between(cudaEvent_t a, cudaEvent_t b) {
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    return ms;
}

// One pipeline call: its arguments, in the order cluster_pipeline initialises them, then the state its steps share.  The
// steps run in order on the context's stream, and the first failure ends the call.
struct Pipeline {
    CallContext &C;
    const float *emb;
    const double *rho;
    size_t N, E, R;
    const double *psi;
    const fa_cluster_config &cfg;
    int32_t *labels, *initial_out;
    double *centroids_out;
    int32_t max_centroids;
    fa_cluster_info *info;
    const int32_t *chunk_index;

    const cudaStream_t s = C.stream;
    const int n = (int)N, e = (int)E, r = (int)R;
    const bool speaker_count =
        cfg.num_speakers != FA_NO_VALUE || cfg.min_speakers != FA_NO_VALUE || cfg.max_speakers != FA_NO_VALUE;
    // the arenas: device, pinned host, and VBx's gamma / pi / ELBOs with the centroids (raw and normalised)
    const float *d_emb32;
    const double *d_rho;
    double *d_emb, *d_train, *d_train_rho, *d_norm, *d_gamma, *d_pi, *d_elbos, *d_cent, *d_cent_n, *h_Z;
    unsigned char *d_ok, *h_ok;
    int *d_idx, *d_init, *d_hard, *d_labels, *d_count, *h_idx, *h_count;
    int32_t *h_init;
    const double *d_tr, *d_tr_rho;   // the training rows
    int Tn = 0;           // training rows: the finite ones, or all when none is (so Tn >= 1)
    int S = 0;            // initial clusters of the cut
    int iterations = 0;   // of VBx
    int detected = 0;     // distinct row-argmax winners of VBx, once counted
    int K = 0;            // centroids
    bool adjusted = false;   // K-Means re-clustered for the speaker count
    float ms_norm = 0, ms_ahc = 0, ms_cut = 0;

    int run() {
        const auto wall0 = std::chrono::steady_clock::now();
        int st = upload_and_filter();
        if (st == FA_OK) st = ahc_and_cut();
        if (st == FA_OK) st = refine();
        if (st == FA_OK) st = apply_speaker_count();
        if (st == FA_OK) st = centroids_and_assign();
        if (st == FA_OK) st = report(wall0);
        return st;
    }

    // 1. Upload, widen to double (:286) and keep the rows with a finite embedding (:591-611); when none is finite, every
    // row trains.
    int upload_and_filter() {
        HostStaging H(true, s);
        int st = H.carve(C.d_buf, [&](HostStaging::Layout &c) {
            d_emb32 = c.in(emb, N * E);
            d_emb = c.take<double>(N * E);
            d_rho = c.in(rho, N * R);
            d_ok = c.take<unsigned char>(N);
            d_idx = c.take<int>(N);               // train idx
            d_train = c.take<double>(N * E);
            d_train_rho = c.take<double>(N * R);
            d_norm = c.take<double>(N * E);       // normalised train
            d_init = c.take<int>(N);              // init labels
            d_hard = c.take<int>(N);
            d_labels = c.take<int>(N);
            d_count = c.take<int>(64);
        }, 4096);
        if (st != FA_OK) return st;
        st = carve_arena(C.h_buf, [&](Carver &c) {
            h_ok = c.take<unsigned char>(N);
            h_idx = c.take<int>(N);
            h_init = c.take<int32_t>(N);
            h_count = c.take<int>(16);
            h_Z = c.take<double>(N > 1 ? (N - 1) * 4 : 4);
        }, 4096);
        if (st != FA_OK) return st;
        st = ahc::launch_widen_rows(d_emb32, d_emb, (long long)N * E, s);
        if (st != FA_OK) return st;
        st = vbx::finite_rows_device(d_emb32, n, e, d_ok, s);
        if (st != FA_OK) return st;
        FA_CUDA_TRY(cudaMemcpyAsync(h_ok, d_ok, N, cudaMemcpyDeviceToHost, s));
        FA_CUDA_TRY(cudaStreamSynchronize(s));
        for (int i = 0; i < n; ++i)
            if (h_ok[i]) h_idx[Tn++] = i;
        if (Tn == 0) {
            for (int i = 0; i < n; ++i) h_idx[i] = i;
            Tn = n;
        }
        d_tr = d_emb;
        d_tr_rho = d_rho;
        if (Tn != n) {
            FA_CUDA_TRY(cudaMemcpyAsync(d_idx, h_idx, Tn * sizeof(int), cudaMemcpyHostToDevice, s));
            st = vbx::gather_rows_device(d_emb, d_idx, Tn, e, d_train, s);
            if (st != FA_OK) return st;
            st = vbx::gather_rows_device(d_rho, d_idx, Tn, r, d_train_rho, s);
            if (st != FA_OK) return st;
            d_tr = d_train;
            d_tr_rho = d_train_rho;
        }
        return FA_OK;
    }

    // 2. AHC on the normalised training rows and the dendrogram cut (:301-309): S initial clusters, labelled 0..S-1.
    int ahc_and_cut() {
        if (Tn >= 2) {
            FA_CUDA_TRY(cudaEventRecord(C.ev[0], s));
            int st = ahc::launch_normalize_rows(d_tr, d_norm, Tn, e, s);
            if (st != FA_OK) return st;
            FA_CUDA_TRY(cudaEventRecord(C.ev[1], s));
            st = C.solver.linkage_device(d_norm, Tn, e, h_Z);
            FA_CUDA_TRY(cudaEventRecord(C.ev[2], s));
            FA_CUDA_TRY(cudaEventSynchronize(C.ev[2]));
            ms_norm = ms_between(C.ev[0], C.ev[1]);
            ms_ahc = ms_between(C.ev[1], C.ev[2]);
            const auto t0 = std::chrono::steady_clock::now();
            if (st == FA_OK) {
                ahc::dendrogram_cut(h_Z, Tn, cfg.threshold, h_init);
            } else if (st == FA_RUNTIME_ERROR || st == FA_UNSUPPORTED) {
                for (int i = 0; i < Tn; ++i) h_init[i] = i;   // AHCClustering.swift:52-55: FFI failure -> identity labels
            } else {
                return st;
            }
            ms_cut = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
        } else {
            for (int i = 0; i < Tn; ++i) h_init[i] = 0;
        }
        for (int i = 0; i < Tn; ++i) S = std::max(S, h_init[i] + 1);   // labels are canonical 0..S-1
        S = std::max(S, 1);
        if (initial_out) {
            for (int i = 0; i < n; ++i) initial_out[i] = -1;
            for (int i = 0; i < Tn; ++i) initial_out[h_idx[i]] = h_init[i];
        }
        return FA_OK;
    }

    // 3. VBx from the initial clusters on the training rows' rho (:311-343).
    int refine() {
        FA_CUDA_TRY(cudaEventRecord(C.ev[3], s));
        FA_CUDA_TRY(cudaMemcpyAsync(d_init, h_init, Tn * sizeof(int), cudaMemcpyHostToDevice, s));
        // arena for gamma / pi / elbos / centroids (depends on S, known only now), at least 1 MB
        const vbx::Config vc = to_vbx(cfg.vbx);
        int st = C.cent_pool.grow((size_t)1 << 20);
        if (st != FA_OK) return st;
        st = carve_arena(C.cent_pool, [&](Carver &c) {
            d_gamma = c.take<double>((size_t)Tn * S);
            d_pi = c.take<double>(S);
            d_elbos = c.take<double>(std::max(vc.max_iterations, 1));
            d_cent = c.take<double>((size_t)S * E + E);
            d_cent_n = c.take<double>((size_t)S * E + E);
        }, 8192);
        if (st != FA_OK) return st;
        std::vector<double> psi_eff(R, 1.0);   // VBxClustering.swift:71-76: identity when psi does not match
        if (psi) std::memcpy(psi_eff.data(), psi, R * sizeof(double));
        return vbx::refine_device(C.vbx_pool, d_tr_rho, Tn, r, psi_eff.data(), d_init, S, vc, d_gamma, d_pi, d_elbos,
                                  d_hard, &iterations, s);
    }

    // VBxOutput.assignedClusterCount: the distinct row-argmax winners among the S speakers.  Their download synchronises
    // the stream.
    int count_winners() {
        std::vector<int> hard(Tn);
        FA_CUDA_TRY(cudaMemcpyAsync(hard.data(), d_hard, sizeof(int) * Tn, cudaMemcpyDeviceToHost, s));
        FA_CUDA_TRY(cudaStreamSynchronize(s));
        std::vector<char> seen(S, 0);
        detected = 0;
        for (const int h : hard)
            if (h >= 0 && h < S && !seen[h]) {
                seen[h] = 1;
                ++detected;
            }
        return FA_OK;
    }

    // 4. Speaker-count constraints (:311-336, VBxClustering.swift:685-733): when VBx's speakers fall outside the resolved
    // bounds, K-Means re-clusters the training rows into the nearest bound.
    int apply_speaker_count() {
        if (!speaker_count) return FA_OK;
        int st = count_winners();
        if (st != FA_OK) return st;
        long long lo = 1, hi = Tn;
        kmeans::resolve_constraints(Tn, cfg.num_speakers, cfg.min_speakers, cfg.max_speakers, &lo, &hi);
        if (detected >= lo && detected <= hi) return FA_OK;
        const int target = (int)(detected < lo ? lo : hi);
        // the arena may have moved: re-carve (gamma / pi are not needed any more on this path)
        st = carve_arena(C.cent_pool, [&](Carver &c) {
            d_cent = c.take<double>((size_t)target * E + E);
            d_cent_n = c.take<double>((size_t)target * E + E);
        }, 8192);
        if (st != FA_OK) return st;
        st = kmeans::cluster_ninit_device(C.vbx_pool, d_tr, Tn, e, target, 100, 10, 0ull, d_hard, d_cent, &K, nullptr, s);
        if (st != FA_OK) return st;
        st = ahc::launch_normalize_rows_keep(d_cent, d_cent_n, K, e, s);   // normalize (:824-860) for the cosine
        if (st != FA_OK) return st;
        adjusted = true;
        return FA_OK;
    }

    // 5. The centroids of the speakers with pi > 1e-7 (:345-353) unless K-Means made them, then every row's assignment
    // (:357-374) and the downloads of the labels and centroids.
    int centroids_and_assign() {
        FA_CUDA_TRY(cudaEventRecord(C.ev[4], s));
        int st;
        if (!adjusted) {
            st = vbx::centroids_device(C.vbx_pool, d_tr, Tn, e, d_gamma, d_pi, S, d_cent, d_cent_n, d_count, s);
            if (st != FA_OK) return st;
            FA_CUDA_TRY(cudaMemcpyAsync(h_count, d_count, sizeof(int), cudaMemcpyDeviceToHost, s));
            FA_CUDA_TRY(cudaStreamSynchronize(s));
            K = *h_count;
        }
        if (K == 0) {
            // Unreachable.  The reference recomputes the centroids from the initial clusters when no speaker has
            // pi > 1e-7, and takes the mean of all embeddings when that leaves none (OfflineDiarizerManager.swift:687-690,
            // :748-786).  Here Tn >= 1, VBx renormalises pi to sum 1 or falls back to 1/S when the sum is not finite, so
            // some pi >= 1/S > 1e-7 for any S whose Tn x S gamma fits in memory; K-Means returns min(target, Tn) >= 1 rows.
            fa::set_error("internal: no centroid after VBx (S = %d, %d training rows)", S, Tn);
            return FA_RUNTIME_ERROR;
        }
        // constrained assignment (:357-369) needs the full N x K score matrix on the host; plain argmax (:371-374) does not
        const bool constrained = chunk_index != nullptr && K > 1 && !adjusted;   // :357-360
        double *d_scores = nullptr;
        if (constrained) {
            st = carve_arena(C.vbx_pool, [&](Carver &c) { d_scores = c.take<double>(N * (size_t)K); }, 1024);
            if (st != FA_OK) return st;
        }
        st = vbx::assign_device(d_emb, n, e, d_cent_n, nullptr, K, d_labels, d_scores, s);
        if (st != FA_OK) return st;
        if (constrained) {
            std::vector<double> h_scores(N * (size_t)K);
            FA_CUDA_TRY(cudaMemcpyAsync(h_scores.data(), d_scores, h_scores.size() * sizeof(double), cudaMemcpyDeviceToHost,
                                        s));
            FA_CUDA_TRY(cudaStreamSynchronize(s));
            assign::constrained_assign(h_scores.data(), (long long)N, K, chunk_index, labels);
        } else {
            FA_CUDA_TRY(cudaMemcpyAsync(labels, d_labels, N * sizeof(int), cudaMemcpyDeviceToHost, s));
        }
        if (centroids_out && max_centroids > 0) {
            const int kc = std::min(K, max_centroids);
            FA_CUDA_TRY(cudaMemcpyAsync(centroids_out, d_cent, (size_t)kc * E * sizeof(double), cudaMemcpyDeviceToHost, s));
        }
        FA_CUDA_TRY(cudaEventRecord(C.ev[5], s));
        return FA_OK;
    }

    // 6. The final synchronisation and the caller's info.  When no speaker count was set, the winners were not counted
    // yet: for the info they are now, and their download is the synchronisation.
    int report(std::chrono::steady_clock::time_point wall0) {
        if (info && !speaker_count) {
            const int st = count_winners();
            if (st != FA_OK) return st;
        } else {
            FA_CUDA_TRY(cudaStreamSynchronize(s));
        }
        if (!info) return FA_OK;
        info->training_count = Tn;
        info->initial_clusters = S;
        info->vbx_iterations = iterations;
        info->centroid_count = K;
        info->ms_normalize = ms_norm;
        info->ms_ahc = ms_ahc;
        info->ms_cut = ms_cut;
        info->ms_vbx = ms_between(C.ev[3], C.ev[4]);
        info->ms_assign = ms_between(C.ev[4], C.ev[5]);
        info->ms_total = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - wall0).count();
        info->was_adjusted = adjusted ? 1 : 0;
        info->detected_clusters = detected;
        return FA_OK;
    }
};

int cluster_pipeline(CallContext &C, const float *emb, const double *rho, size_t N, size_t E, size_t R,
                     const double *psi, const fa_cluster_config &cfg, int32_t *labels, int32_t *initial_out,
                     double *centroids_out, int32_t max_centroids, fa_cluster_info *info, const int32_t *chunk_index) {
    return Pipeline{C, emb, rho, N, E, R, psi, cfg, labels, initial_out, centroids_out, max_centroids, info, chunk_index}
        .run();
}

// Independent sets run on disjoint SM partitions: `lanes` host threads, each leasing a context whose merge kernel is
// capped at (SMs / lanes) - 1 worker CTAs, pull sets from a shared counter.
int cluster_batch(const float *emb, const double *rho, const int64_t *set_offsets, int32_t set_count, size_t emb_dim,
                  size_t rho_dim, const double *psi, const fa_cluster_config &cfg, const int32_t *chunk_index,
                  int32_t *labels, fa_cluster_info *infos) {
    int dev = 0;
    FA_CUDA_TRY(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    FA_CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
    // Concurrency: see ahc::plan_batch_lanes
    long long n_max = 0;
    for (int m = 0; m < set_count; ++m) n_max = std::max<long long>(n_max, set_offsets[m + 1] - set_offsets[m]);
    const ahc::BatchLanes plan = ahc::plan_batch_lanes(set_count, n_max, (int)emb_dim, prop.multiProcessorCount);
    const int lanes = plan.lanes, worker_limit = plan.worker_limit;
    std::atomic<int> next{0};
    std::vector<int> status(lanes, FA_OK);
    std::vector<std::array<char, 512>> messages(lanes);   // a failed lane's error text, empty when it set none
    // Each lane is a plain std::thread: nothing may escape it (an exception leaving a thread function is std::terminate),
    // so run_guarded turns every failure, exceptions included, into status[] and the lane's own error text.
    auto run = [&](int lane) noexcept {
        const unsigned serial = error_serial();
        status[lane] = run_guarded([&]() -> int {
            const cudaError_t e = cudaSetDevice(dev);
            if (e != cudaSuccess) return cuda_failure(e, "cudaSetDevice", __FILE__, __LINE__);
            return with_context(worker_limit, [&](CallContext &C) {
                for (;;) {
                    const int m = next.fetch_add(1);
                    if (m >= set_count) return (int)FA_OK;
                    const int64_t a = set_offsets[m], b = set_offsets[m + 1];
                    if (b == a) continue;   // not clustered: the caller zeroed its info
                    const int st = cluster_pipeline(C, emb + (size_t)a * emb_dim, rho + (size_t)a * rho_dim,
                                                    (size_t)(b - a), emb_dim, rho_dim, psi, cfg, labels + a, nullptr,
                                                    nullptr, 0, infos ? infos + m : nullptr,
                                                    chunk_index ? chunk_index + a : nullptr);
                    if (st != FA_OK) return st;
                }
            });
        });
        if (status[lane] != FA_OK && error_serial() != serial)
            std::snprintf(messages[lane].data(), messages[lane].size(), "%s", fa::last_error());
        if (status[lane] != FA_OK) next.store(set_count);   // the other lanes stop taking new sets
    };
    // Lane 0 runs on the calling thread.  Every thread that starts is joined below: nothing between its start and the
    // join can throw (the vector is reserved, and run is noexcept).
    std::vector<std::thread> threads;
    threads.reserve(lanes);
    try {
        for (int l = 1; l < lanes; ++l) threads.emplace_back(run, l);
    } catch (...) {   // std::system_error: run with the lanes that did start
    }
    run(0);
    for (auto &t : threads) t.join();
    for (int l = 0; l < lanes; ++l)
        if (status[l] != FA_OK) {
            if (messages[l][0]) fa::set_error("%s", messages[l].data());
            return status[l];
        }
    return FA_OK;
}

int l2_normalize_rows(CallContext &C, const double *x, size_t rows, size_t dim, double *out) {
    HostStaging H(true, C.stream);
    const double *d_in;
    double *d_out;
    int st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_in = l.in(x, rows * dim);
        d_out = l.out(out, rows * dim);
    }, 512);
    if (st != FA_OK) return st;
    st = ahc::launch_normalize_rows(d_in, d_out, (int)rows, (int)dim, C.stream);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

// AHCClustering.cluster (AHCClustering.swift:20-67) for count >= 2 and dim >= 1
int ahc_cluster(CallContext &C, const double *features, size_t count, size_t dim, double threshold, int32_t *labels) {
    HostStaging H(true, C.stream);
    const double *d_in;
    double *d_norm, *h_Z;
    int st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_in = l.in(features, count * dim);
        d_norm = l.take<double>(count * dim);
    }, 512);
    if (st != FA_OK) return st;
    st = carve_arena(C.h_buf, [&](Carver &c) { h_Z = c.take<double>((count - 1) * 4); }, 512);
    if (st != FA_OK) return st;
    st = ahc::launch_normalize_rows(d_in, d_norm, (int)count, (int)dim, C.stream);
    if (st != FA_OK) return st;
    st = C.solver.linkage_device(d_norm, (int)count, (int)dim, h_Z);
    if (st == FA_RUNTIME_ERROR || st == FA_UNSUPPORTED) {      // FFI failure -> Array(0..<count) (:52-55)
        for (size_t i = 0; i < count; ++i) labels[i] = (int32_t)i;
        return FA_OK;
    }
    if (st != FA_OK) return st;
    ahc::dendrogram_cut(h_Z, (long long)count, threshold, labels);
    return FA_OK;
}

// KMeansClustering.clusterWithCentroidsNInit for N >= 1, D >= 1 and num_clusters >= 1: min(num_clusters, N) centroid rows
int kmeans_cluster(CallContext &C, const double *emb, size_t N, size_t D, int32_t num_clusters, int32_t max_iterations,
                   int32_t n_init, uint64_t base_seed, int32_t *labels, double *centroids, int32_t *centroid_rows,
                   int32_t *best_init) {
    const size_t rows_needed = std::min<size_t>((size_t)num_clusters, N);
    HostStaging H(true, C.stream);
    const double *d_emb;
    double *d_cent;
    int *d_labels;
    int st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_emb = l.in(emb, N * D);
        d_cent = l.out(centroids, rows_needed * D);
        d_labels = l.out(labels, N);
    }, 1024);
    if (st != FA_OK) return st;
    int rows = 0, best = 0;
    st = kmeans::cluster_ninit_device(C.vbx_pool, d_emb, (int)N, (int)D, num_clusters, max_iterations, n_init, base_seed,
                                      d_labels, d_cent, &rows, &best, C.stream);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(H.back(labels, d_labels, N));
    FA_CUDA_TRY(H.back(centroids, d_cent, (size_t)rows * D));   // the rows K-Means returned
    FA_CUDA_TRY(H.sync());
    if (centroid_rows) *centroid_rows = rows;
    if (best_init) *best_init = best;
    return FA_OK;
}

int vbx_refine(CallContext &C, const double *rho, size_t T, size_t D, const double *psi, size_t psi_len,
               const int32_t *initial, int32_t S, const fa_vbx_config &cfg, double *gamma, double *pi, double *elbos,
               int32_t *hard, int32_t *iterations) {
    const int cap = std::max(cfg.max_iterations, 1);
    HostStaging H(true, C.stream);
    const double *d_x;
    const int *d_init;
    double *d_gamma, *d_pi, *d_elbos;
    int *d_hard;
    int st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_x = l.in(rho, T * D);
        d_init = l.in(initial, T);
        d_gamma = l.out(gamma, T * (size_t)S);
        d_pi = l.out(pi, S);
        d_elbos = l.out(elbos, cap);
        d_hard = l.out(hard, T);
    }, 1024);
    if (st != FA_OK) return st;
    std::vector<double> psi_eff(D, 1.0);
    if (psi && psi_len == D) std::memcpy(psi_eff.data(), psi, D * sizeof(double));
    int its = 0;
    st = vbx::refine_device(C.vbx_pool, d_x, (int)T, (int)D, psi_eff.data(), d_init, S, to_vbx(cfg), d_gamma, d_pi, d_elbos,
                            d_hard, &its, C.stream);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(H.finish());
    if (iterations) *iterations = its;
    return FA_OK;
}

int compute_centroids(CallContext &C, const double *emb, size_t T, size_t dim, const double *gamma, const double *pi,
                      int32_t S, double *centroids, int32_t *centroid_count) {
    HostStaging H(true, C.stream);
    const double *d_emb, *d_gamma, *d_pi;
    double *d_cent, *d_cent_n;
    int *d_count;
    int st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_emb = l.in(emb, T * dim);
        d_gamma = l.in(gamma, T * (size_t)S);
        d_pi = l.in(pi, S);
        d_cent = l.out(centroids, (size_t)S * dim);
        d_cent_n = l.take<double>((size_t)S * dim);
        d_count = l.take<int>(64);
    }, 1024);
    if (st != FA_OK) return st;
    st = vbx::centroids_device(C.vbx_pool, d_emb, (int)T, (int)dim, d_gamma, d_pi, S, d_cent, d_cent_n, d_count, C.stream);
    if (st != FA_OK) return st;
    int K = 0;
    FA_CUDA_TRY(cudaMemcpyAsync(&K, d_count, sizeof(int), cudaMemcpyDeviceToHost, C.stream));
    FA_CUDA_TRY(cudaStreamSynchronize(C.stream));
    *centroid_count = K;
    if (K > 0) {   // the centroids of the K speakers kept
        FA_CUDA_TRY(H.back(centroids, d_cent, (size_t)K * dim));
        FA_CUDA_TRY(H.sync());
    }
    return FA_OK;
}

// OfflineDiarizerManager.assignEmbeddings (:789-883) for N >= 1 and K >= 1
int assign_embeddings(CallContext &C, const double *emb, size_t N, size_t dim, const double *centroids, int32_t K,
                      int32_t *labels, double *scores) {
    HostStaging H(true, C.stream);
    const double *d_emb, *d_craw;
    double *d_cn, *d_scores;
    int *d_labels;
    int st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_emb = l.in(emb, N * dim);
        d_craw = l.in(centroids, (size_t)K * dim);
        d_cn = l.take<double>((size_t)K * dim);
        d_labels = l.out(labels, N);
        d_scores = l.out(scores, N * (size_t)K);
    }, 1024);
    if (st != FA_OK) return st;
    // centroid normalisation (:793, :824-860; zero rows kept) with the same kernel the pipeline uses
    st = ahc::launch_normalize_rows_keep(d_craw, d_cn, K, (int)dim, C.stream);
    if (st != FA_OK) return st;
    st = vbx::assign_device(d_emb, (int)N, (int)dim, d_cn, nullptr, K, d_labels, d_scores, C.stream);
    if (st != FA_OK) return st;
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

} // namespace fa
