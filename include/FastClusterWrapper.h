/* Drop-in declaration of the reference's only C boundary on the clustering path.
 *
 * Replaces Sources/FastClusterWrapper/include/FastClusterWrapper.h:11-40 of FluidAudio: same symbol, same status
 * values, same buffer contract, so AHCClustering.swift:40-50 links against libfluidaudio_b200.so unchanged
 * (module map: swift/FastClusterWrapper/module.modulemap).  The body runs on an sm_90a GPU; there is no CPU
 * fallback — without a device the call returns FASTCLUSTER_WRAPPER_RUNTIME_ERROR, which the Swift caller already
 * maps to "every point its own cluster" (AHCClustering.swift:52-55).
 */
#ifndef FASTCLUSTER_WRAPPER_H
#define FASTCLUSTER_WRAPPER_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    FASTCLUSTER_WRAPPER_SUCCESS = 0,
    FASTCLUSTER_WRAPPER_INVALID_ARGUMENT = 1,   /* NULL buffer, or dimension == 0 with pointCount > 0 */
    FASTCLUSTER_WRAPPER_INDEX_OVERFLOW = 2,     /* pointCount or dimension > INT32_MAX */
    FASTCLUSTER_WRAPPER_OUTPUT_TOO_SMALL = 3,   /* dendrogramLength < 4 * (pointCount - 1) */
    FASTCLUSTER_WRAPPER_ALLOCATION_FAILURE = 4, /* host or device allocation failed */
    FASTCLUSTER_WRAPPER_RUNTIME_ERROR = 5,      /* NaN distance, CUDA failure, no device */
    FASTCLUSTER_WRAPPER_UNKNOWN_ERROR = 255
} fastcluster_wrapper_status;

/* Centroid-linkage dendrogram of `pointCount` row-major vectors of `dimension` doubles (host memory, already
 * L2-normalised by the caller).  Writes (pointCount - 1) rows of (smaller id, larger id, distance, size) in merge
 * order; row m is node id pointCount + m.  pointCount == 0 or 1 writes nothing and succeeds.  Synchronous,
 * re-entrant, keeps no pointer after returning. */
fastcluster_wrapper_status fastcluster_compute_centroid_linkage(const double *data, size_t pointCount,
                                                                size_t dimension, double *dendrogramOut,
                                                                size_t dendrogramLength);

#ifdef __cplusplus
}
#endif
#endif /* FASTCLUSTER_WRAPPER_H */
