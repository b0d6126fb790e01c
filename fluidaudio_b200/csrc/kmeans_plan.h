// Host entry points of the speaker-count-constrained K-Means re-clustering (kmeans_kernels.cu).
#pragma once

#include "fa_common.cuh"
#include <cuda_runtime.h>

namespace fa {
namespace kmeans {

// KMeansClustering.clusterWithCentroidsNInit on device-resident raw embeddings d_emb [N x D] (row-major doubles).
// d_labels [N] and d_centroids [min(k, N) x D] receive the winning run; *rows the number of centroid rows,
// *best_init the index of the winning seed.  Scratch comes from `pool`.
int cluster_ninit_device(DeviceBuffer<> &pool, const double *d_emb, int N, int D, int num_clusters, int max_iterations,
                         int n_init, unsigned long long base_seed, int *d_labels, double *d_centroids, int *rows,
                         int *best_init, cudaStream_t stream);

// SpeakerCountConstraints.resolve; absent options are FA_NO_VALUE (INT32_MIN).
void resolve_constraints(long long num_embeddings, long long num_speakers, long long min_speakers, long long max_speakers,
                         long long *lo, long long *hi);

} // namespace kmeans
} // namespace fa
