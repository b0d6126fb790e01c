// Host side of the clustering entry points (cluster_pipeline.cu): the diarization pipeline with its batch lanes, and the
// standalone stages, each on a leased call context (call_context.h).  Data pointers are host pointers, arguments checked
// by the C ABI.
#pragma once

#include "../../include/fluidaudio_b200.h"
#include "call_context.h"

namespace fa {

// OfflineDiarizerManager.cluster(_:) :286-375 on one context; chunk_index selects the constrained assignment
int cluster_pipeline(CallContext &C, const float *emb, const double *rho, size_t N, size_t E, size_t R,
                     const double *psi, const fa_cluster_config &cfg, int32_t *labels, int32_t *initial_out,
                     double *centroids_out, int32_t max_centroids, fa_cluster_info *info, const int32_t *chunk_index);
// the pipeline over every non-empty set, on concurrent lanes of the current device
int cluster_batch(const float *emb, const double *rho, const int64_t *set_offsets, int32_t set_count, size_t emb_dim,
                  size_t rho_dim, const double *psi, const fa_cluster_config &cfg, const int32_t *chunk_index,
                  int32_t *labels, fa_cluster_info *infos);

// the stages behind fa_l2_normalize_rows, fa_ahc_cluster, fa_kmeans_cluster, fa_vbx_refine, fa_compute_centroids and
// fa_assign_embeddings, for the inputs those leave to the device
int l2_normalize_rows(CallContext &C, const double *x, size_t rows, size_t dim, double *out);
int ahc_cluster(CallContext &C, const double *features, size_t count, size_t dim, double threshold, int32_t *labels);
int kmeans_cluster(CallContext &C, const double *emb, size_t N, size_t D, int32_t num_clusters, int32_t max_iterations,
                   int32_t n_init, uint64_t base_seed, int32_t *labels, double *centroids, int32_t *centroid_rows,
                   int32_t *best_init);
int vbx_refine(CallContext &C, const double *rho, size_t T, size_t D, const double *psi, size_t psi_len,
               const int32_t *initial, int32_t S, const fa_vbx_config &cfg, double *gamma, double *pi, double *elbos,
               int32_t *hard, int32_t *iterations);
int compute_centroids(CallContext &C, const double *emb, size_t T, size_t dim, const double *gamma, const double *pi,
                      int32_t S, double *centroids, int32_t *centroid_count);
int assign_embeddings(CallContext &C, const double *emb, size_t N, size_t dim, const double *centroids, int32_t K,
                      int32_t *labels, double *scores);

} // namespace fa
