// Host entry points of the VBx / centroid / assignment kernels (vbx_kernels.cu).
#pragma once

#include "fa_common.cuh"
#include <cuda_runtime.h>

namespace fa {
namespace vbx {

struct Config {
    double Fa = 0.07;            // OfflineDiarizerConfig.Clustering.community.warmStartFa
    double Fb = 0.8;             // warmStartFb
    int max_iterations = 20;     // OfflineDiarizerConfig.VBx.community
    double epsilon = 1e-4;
    double init_smoothing = 7.0; // VBxClustering.swift:131
};

// Opts the kernels below that take more than 48 KB of dynamic shared memory in to their maxima.  A function attribute
// holds for the device current when it is set: call it on every device the kernels run on.
int set_smem_limits();

// `pool`: the scratch arena, reused across calls (grown on demand).
int refine_device(DeviceBuffer<> &pool, const double *d_x, int T, int D, const double *h_psi, const int *d_init, int S,
                  const Config &cfg, double *d_gamma, double *d_pi, double *d_elbos, int *d_hard, int *iterations_host,
                  cudaStream_t stream);
int centroids_device(DeviceBuffer<> &pool, const double *d_emb, int T, int E, const double *d_gamma, const double *d_pi,
                     int S, double *d_cent, double *d_cent_n, int *d_count, cudaStream_t stream);
int assign_device(const double *d_emb, int N, int E, const double *d_cent_n, const int *d_count, int K_fixed,
                  int *d_labels, double *d_scores, cudaStream_t stream);
int finite_rows_device(const float *d_emb, int N, int E, unsigned char *d_ok, cudaStream_t stream);
int gather_rows_device(const double *d_src, const int *d_idx, int rows, int dim, double *d_dst, cudaStream_t stream);

} // namespace vbx
} // namespace fa
