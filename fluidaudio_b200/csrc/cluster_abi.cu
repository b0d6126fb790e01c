// C ABI of the clustering backend (declared in include/fluidaudio_b200.h and include/FastClusterWrapper.h): AHC, VBx,
// K-Means, assignment and reconstruction, and the cluster pipeline (cluster_pipeline.cu) with its batch lanes.  Every
// entry point that returns a status returns through guard() (c_abi.h); the device calls lease the pooled call context.
#include "../../include/FastClusterWrapper.h"
#include "c_abi.h"

#include "ahc_plan.h"
#include "assign_host.h"
#include "call_context.h"
#include "cluster_plan.h"
#include "kmeans_plan.h"
#include "reconstruct_host.h"

#include <algorithm>
#include <vector>

using namespace fa;

static fastcluster_wrapper_status to_fc(int st) {
    switch (st) {
    case FA_OK: return FASTCLUSTER_WRAPPER_SUCCESS;
    case FA_INVALID_ARGUMENT: return FASTCLUSTER_WRAPPER_INVALID_ARGUMENT;
    case FA_INDEX_OVERFLOW: return FASTCLUSTER_WRAPPER_INDEX_OVERFLOW;
    case FA_OUTPUT_TOO_SMALL: return FASTCLUSTER_WRAPPER_OUTPUT_TOO_SMALL;
    case FA_ALLOCATION_FAILURE: return FASTCLUSTER_WRAPPER_ALLOCATION_FAILURE;
    case FA_UNKNOWN_ERROR: return FASTCLUSTER_WRAPPER_UNKNOWN_ERROR;
    default: return FASTCLUSTER_WRAPPER_RUNTIME_ERROR;   // NaN, CUDA failure, no device, unsupported size
    }
}

FA_API fastcluster_wrapper_status fastcluster_compute_centroid_linkage(const double *data, size_t pointCount,
                                                                       size_t dimension, double *dendrogramOut,
                                                                       size_t dendrogramLength) {
    return to_fc(guard(__func__, [&]() -> int {
        // argument contract first, exactly as FastClusterWrapper.cpp:203-223 (no device needed for these)
        if (data == nullptr || dendrogramOut == nullptr) return FA_INVALID_ARGUMENT;
        if (pointCount == 0) return FA_OK;
        if (dimension == 0) return FA_INVALID_ARGUMENT;
        if (pointCount > 0x7fffffffull || dimension > 0x7fffffffull) return FA_INDEX_OVERFLOW;
        const size_t need = pointCount > 1 ? (pointCount - 1) * 4 : 0;
        if (dendrogramLength < need) return FA_OUTPUT_TOO_SMALL;
        if (pointCount == 1) return FA_OK;
        if (require_device() != FA_OK) return FA_NO_DEVICE;
        return with_context(0, [&](CallContext &C) {
            return C.solver.linkage_host(data, pointCount, dimension, dendrogramOut, dendrogramLength);
        });
    }));
}

FA_API void fa_ahc_last_stage_ms(float *out4) {
    if (!out4) return;
    const float *m = ahc::last_stage_ms();
    for (int q = 0; q < 4; ++q) out4[q] = m[q];
}

FA_API fa_status fa_l2_normalize_rows(const double *x, size_t rows, size_t dim, double *out) {
    return guard(__func__, [&]() -> int {
        if (!x || !out) return FA_STATUS_INVALID_ARGUMENT;
        if (rows == 0 || dim == 0) return FA_STATUS_OK;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) { return l2_normalize_rows(C, x, rows, dim, out); });
    });
}

FA_API fa_status fa_dendrogram_cut(const double *Z, size_t count, double threshold, int32_t *labels) {
    return guard(__func__, [&]() -> int {
        if ((!Z && count > 1) || (!labels && count > 0)) return FA_STATUS_INVALID_ARGUMENT;
        ahc::dendrogram_cut(Z, (long long)count, threshold, labels);
        return FA_STATUS_OK;
    });
}

// AHCClustering.cluster (AHCClustering.swift:20-67)
FA_API fa_status fa_ahc_cluster(const double *features, size_t count, size_t dim, double threshold, int32_t *labels) {
    return guard(__func__, [&]() -> int {
        if (count == 0) return FA_STATUS_OK;                       // guard count > 0 else []
        if (!labels) return FA_STATUS_INVALID_ARGUMENT;
        if (dim == 0) {                                            // zero-dimension vectors: all cluster 0 (:26-28)
            for (size_t i = 0; i < count; ++i) labels[i] = 0;
            return FA_STATUS_OK;
        }
        if (!features) return FA_STATUS_INVALID_ARGUMENT;
        if (count == 1) {
            labels[0] = 0;
            return FA_STATUS_OK;
        }
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) { return ahc_cluster(C, features, count, dim, threshold, labels); });
    });
}

FA_API void fa_vbx_default_config(fa_vbx_config *cfg) {
    if (!cfg) return;
    cfg->Fa = 0.07;
    cfg->Fb = 0.8;
    cfg->max_iterations = 20;
    cfg->epsilon = 1e-4;
    cfg->init_smoothing = 7.0;
}

FA_API void fa_cluster_default_config(fa_cluster_config *cfg) {
    if (!cfg) return;
    cfg->threshold = 0.6;
    fa_vbx_default_config(&cfg->vbx);
    cfg->num_speakers = cfg->min_speakers = cfg->max_speakers = FA_NO_VALUE;
    cfg->reserved = 0;
}

FA_API void fa_reconstruct_default_config(fa_reconstruct_config *cfg) {
    if (!cfg) return;
    const reconstruct::Config d;
    cfg->frame_duration = d.frame_duration;
    cfg->window_duration = d.window_duration;
    cfg->min_gap_duration = d.min_gap_duration;
    cfg->seg_min_duration_off = d.seg_min_duration_off;
    cfg->seg_min_duration_on = d.seg_min_duration_on;
    cfg->min_segment_duration = d.min_segment_duration;
    cfg->exclusive_segments = d.exclusive_segments ? 1 : 0;
    cfg->reserved = 0;
}

FA_API fa_status fa_build_segments(const float *weights, int32_t num_chunks, int32_t num_frames, int32_t num_speakers,
                                   const double *chunk_offsets, int32_t offsets_count, const int32_t *hard_clusters,
                                   int32_t hard_rows, int32_t centroid_count, const fa_reconstruct_config *cfg,
                                   int32_t *seg_cluster, float *seg_start, float *seg_end, float *seg_quality,
                                   int32_t segment_cap, int32_t *segment_count) {
    return guard(__func__, [&]() -> int {
        if (!cfg || !segment_count || num_speakers < 0 || offsets_count < 0 || hard_rows < 0 || segment_cap < 0 ||
            (num_chunks > 0 && num_frames > 0 && num_speakers > 0 && !weights) || (offsets_count > 0 && !chunk_offsets) ||
            (hard_rows > 0 && !hard_clusters))
            return FA_STATUS_INVALID_ARGUMENT;
        reconstruct::Config c;
        c.frame_duration = cfg->frame_duration;
        c.window_duration = cfg->window_duration;
        c.min_gap_duration = cfg->min_gap_duration;
        c.seg_min_duration_off = cfg->seg_min_duration_off;
        c.seg_min_duration_on = cfg->seg_min_duration_on;
        c.min_segment_duration = cfg->min_segment_duration;
        c.exclusive_segments = cfg->exclusive_segments != 0;
        std::vector<reconstruct::Segment> segs;
        reconstruct::build_segments(weights, num_chunks, num_frames, num_speakers, chunk_offsets, offsets_count,
                                    hard_clusters, hard_rows, centroid_count, c, segs);
        *segment_count = (int32_t)segs.size();
        const int32_t n = std::min<int32_t>((int32_t)segs.size(), segment_cap);
        for (int32_t i = 0; i < n; ++i) {
            if (seg_cluster) seg_cluster[i] = segs[i].cluster;
            if (seg_start) seg_start[i] = segs[i].start;
            if (seg_end) seg_end[i] = segs[i].end;
            if (seg_quality) seg_quality[i] = segs[i].quality;
        }
        return (int32_t)segs.size() > segment_cap ? FA_STATUS_OUTPUT_TOO_SMALL : FA_STATUS_OK;
    });
}

FA_API fa_status fa_build_speaker_database(const int32_t *seg_cluster, int32_t segment_count, const double *centroids,
                                           int32_t K, int32_t dim, float *database, int32_t *segment_counts) {
    return guard(__func__, [&]() -> int {
        if (segment_count < 0 || K < 0 || dim < 0 || (segment_count > 0 && !seg_cluster) ||
            (K > 0 && (!segment_counts || (dim > 0 && (!centroids || !database)))))
            return FA_STATUS_INVALID_ARGUMENT;
        reconstruct::build_speaker_database(seg_cluster, segment_count, centroids, K, dim, database, segment_counts);
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_speaker_constraints_resolve(int64_t num_embeddings, int64_t num_speakers, int64_t min_speakers,
                                                int64_t max_speakers, int64_t *resolved_min, int64_t *resolved_max) {
    return guard(__func__, [&]() -> int {
        if (!resolved_min || !resolved_max) return FA_STATUS_INVALID_ARGUMENT;
        long long lo = 0, hi = 0;
        kmeans::resolve_constraints(num_embeddings, num_speakers, min_speakers, max_speakers, &lo, &hi);
        *resolved_min = lo;
        *resolved_max = hi;
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_kmeans_cluster(const double *emb, size_t N, size_t D, int32_t num_clusters, int32_t max_iterations,
                                   int32_t n_init, uint64_t base_seed, int32_t *labels, double *centroids,
                                   int32_t centroid_cap, int32_t *centroid_rows, int32_t *best_init) {
    return guard(__func__, [&]() -> int {
        if (centroid_rows) *centroid_rows = 0;
        if (best_init) *best_init = 0;
        if (N == 0) return FA_STATUS_OK;                                  // :50-52
        if (!emb || !labels || max_iterations < 0) return FA_STATUS_INVALID_ARGUMENT;
        const long long rows_needed = D == 0 || num_clusters <= 0 ? 0 : std::min<long long>(num_clusters, (long long)N);
        if (rows_needed > 0 && (!centroids || centroid_cap < rows_needed)) return FA_STATUS_OUTPUT_TOO_SMALL;
        if (rows_needed == 0) {                                           // :53-58: dimension 0 or k <= 0 -> all zeros
            for (size_t i = 0; i < N; ++i) labels[i] = 0;
            return FA_STATUS_OK;
        }
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) {
            return kmeans_cluster(C, emb, N, D, num_clusters, max_iterations, n_init, base_seed, labels, centroids,
                                  centroid_rows, best_init);
        });
    });
}

FA_API fa_status fa_vbx_refine(const double *rho, size_t T, size_t D, const double *psi, size_t psi_len,
                               const int32_t *initial, int32_t S, const fa_vbx_config *cfg, double *gamma, double *pi,
                               double *elbos, int32_t *hard, int32_t *iterations) {
    return guard(__func__, [&]() -> int {
        if (!rho || !cfg || !gamma || !pi || !elbos || !hard || T == 0 || D == 0 || S <= 0)
            return FA_STATUS_INVALID_ARGUMENT;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) {
            return vbx_refine(C, rho, T, D, psi, psi_len, initial, S, *cfg, gamma, pi, elbos, hard, iterations);
        });
    });
}

FA_API fa_status fa_compute_centroids(const double *emb, size_t T, size_t dim, const double *gamma, const double *pi,
                                      int32_t S, double *centroids, int32_t *centroid_count) {
    return guard(__func__, [&]() -> int {
        if (!emb || !gamma || !pi || !centroids || !centroid_count || T == 0 || dim == 0 || S <= 0)
            return FA_STATUS_INVALID_ARGUMENT;
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) {
            return compute_centroids(C, emb, T, dim, gamma, pi, S, centroids, centroid_count);
        });
    });
}

FA_API fa_status fa_assign_embeddings(const double *emb, size_t N, size_t dim, const double *centroids, int32_t K,
                                      int32_t *labels, double *scores) {
    return guard(__func__, [&]() -> int {
        if (N == 0) return FA_STATUS_OK;
        if (!emb || !labels || dim == 0 || (K > 0 && !centroids)) return FA_STATUS_INVALID_ARGUMENT;
        if (K <= 0) {   // guard !centroids.isEmpty else all zeros (:805-807)
            for (size_t i = 0; i < N; ++i) labels[i] = 0;
            return FA_STATUS_OK;
        }
        if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
        return with_context(0, [&](CallContext &C) {
            return assign_embeddings(C, emb, N, dim, centroids, K, labels, scores);
        });
    });
}

static int diarize_cluster(const float *emb256, const double *rho, size_t N, size_t emb_dim, size_t rho_dim,
                           const double *psi, const fa_cluster_config *cfg, const int32_t *chunk_index, int32_t *labels,
                           int32_t *initial, double *centroids, int32_t max_centroids, fa_cluster_info *info) {
    if (!emb256 || !rho || !cfg || !labels || N == 0 || emb_dim == 0 || rho_dim == 0)
        return refuse("fa_diarize_cluster: null or empty input (the reference throws noSpeechDetected for N == 0)");
    if (N > 0x7fffffffull / 4) return FA_STATUS_INDEX_OVERFLOW;
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return with_context(0, [&](CallContext &C) {
        return cluster_pipeline(C, emb256, rho, N, emb_dim, rho_dim, psi, *cfg, labels, initial, centroids, max_centroids,
                                info, chunk_index);
    });
}

FA_API fa_status fa_diarize_cluster(const float *emb256, const double *rho, size_t N, size_t emb_dim, size_t rho_dim,
                                    const double *psi, const fa_cluster_config *cfg, int32_t *labels, int32_t *initial,
                                    double *centroids, int32_t max_centroids, fa_cluster_info *info) {
    return guard(__func__, [&] {
        return diarize_cluster(emb256, rho, N, emb_dim, rho_dim, psi, cfg, nullptr, labels, initial, centroids,
                               max_centroids, info);
    });
}

FA_API fa_status fa_diarize_cluster_chunks(const float *emb256, const double *rho, size_t N, size_t emb_dim,
                                           size_t rho_dim, const double *psi, const fa_cluster_config *cfg,
                                           const int32_t *chunk_index, int32_t *labels, int32_t *initial,
                                           double *centroids, int32_t max_centroids, fa_cluster_info *info) {
    return guard(__func__, [&] {
        return diarize_cluster(emb256, rho, N, emb_dim, rho_dim, psi, cfg, chunk_index, labels, initial, centroids,
                               max_centroids, info);
    });
}

FA_API fa_status fa_hungarian_solve(const int64_t *cost, int32_t n, int32_t *assignment) {
    return guard(__func__, [&]() -> int {
        if (n < 0 || (n > 0 && (!cost || !assignment))) return FA_STATUS_INVALID_ARGUMENT;
        assign::min_cost_matching(cost, n, assignment);
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_max_score_assignment(const double *scores, int32_t rows, int32_t cols, int32_t *assignment) {
    return guard(__func__, [&]() -> int {
        if (rows < 0 || cols < 0 || (rows > 0 && !assignment) || (rows > 0 && cols > 0 && !scores))
            return FA_STATUS_INVALID_ARGUMENT;
        assign::max_score_matching(scores, rows, cols, assignment);
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_constrained_assign(const double *scores, size_t N, int32_t K, const int32_t *chunk_index,
                                       int32_t *labels) {
    return guard(__func__, [&]() -> int {
        if (N == 0) return FA_STATUS_OK;
        if (!chunk_index || !labels || K < 0 || (K > 0 && !scores)) return FA_STATUS_INVALID_ARGUMENT;
        assign::constrained_assign(scores, (long long)N, K, chunk_index, labels);
        return FA_STATUS_OK;
    });
}

FA_API fa_status fa_build_chunk_assignments(const int32_t *chunk_index, const int32_t *speaker_index,
                                            const int32_t *assignments, size_t N, int32_t num_chunks,
                                            int32_t num_speakers, int32_t cluster_count, int32_t *matrix) {
    return guard(__func__, [&]() -> int {
        if (num_chunks < 0 || num_speakers < 0 || (!matrix && (size_t)num_chunks * num_speakers > 0) ||
            (N > 0 && (!chunk_index || !speaker_index || !assignments)))
            return FA_STATUS_INVALID_ARGUMENT;
        assign::build_chunk_assignments(chunk_index, speaker_index, assignments, (long long)N, num_chunks, num_speakers,
                                        cluster_count, matrix);
        return FA_STATUS_OK;
    });
}

// The batch's argument checks; its lanes are cluster_batch (cluster_pipeline.cu).
static int cluster_batch_impl(const float *emb256, const double *rho, const int64_t *set_offsets, int32_t set_count,
                              size_t emb_dim, size_t rho_dim, const double *psi, const fa_cluster_config *cfg,
                              const int32_t *chunk_index, int32_t *labels, fa_cluster_info *infos) {
    if (!emb256 || !rho || !set_offsets || !cfg || !labels || set_count < 0 || emb_dim == 0 || rho_dim == 0)
        return FA_STATUS_INVALID_ARGUMENT;
    if (set_count == 0) return FA_STATUS_OK;
    if (set_offsets[0] < 0)
        return refuse("fa_diarize_cluster_batch: set_offsets[0] = %lld is negative", (long long)set_offsets[0]);
    for (int m = 0; m < set_count; ++m)
        if (set_offsets[m + 1] < set_offsets[m])
            return refuse("fa_diarize_cluster_batch: set_offsets decrease at set %d (%lld -> %lld)", m,
                          (long long)set_offsets[m], (long long)set_offsets[m + 1]);
    if (infos)   // an empty set is not clustered: its info reads all zeros
        for (int m = 0; m < set_count; ++m)
            if (set_offsets[m + 1] == set_offsets[m]) infos[m] = fa_cluster_info{};
    if (require_device() != FA_OK) return FA_STATUS_NO_DEVICE;
    return cluster_batch(emb256, rho, set_offsets, set_count, emb_dim, rho_dim, psi, *cfg, chunk_index, labels, infos);
}

FA_API fa_status fa_diarize_cluster_batch(const float *emb256, const double *rho, const int64_t *set_offsets,
                                          int32_t set_count, size_t emb_dim, size_t rho_dim, const double *psi,
                                          const fa_cluster_config *cfg, int32_t *labels, fa_cluster_info *infos) {
    return guard(__func__, [&] {
        return cluster_batch_impl(emb256, rho, set_offsets, set_count, emb_dim, rho_dim, psi, cfg, nullptr, labels,
                                  infos);
    });
}

// The reference's default (constrained) assignment per set: chunk_index[row] = TimedEmbedding.chunkIndex of that row,
// numbered inside its own set.
FA_API fa_status fa_diarize_cluster_batch_chunks(const float *emb256, const double *rho, const int64_t *set_offsets,
                                                 int32_t set_count, size_t emb_dim, size_t rho_dim, const double *psi,
                                                 const fa_cluster_config *cfg, const int32_t *chunk_index,
                                                 int32_t *labels, fa_cluster_info *infos) {
    return guard(__func__, [&] {
        return cluster_batch_impl(emb256, rho, set_offsets, set_count, emb_dim, rho_dim, psi, cfg, chunk_index, labels,
                                  infos);
    });
}
