"""Clustering on a second device of the same process (run with ``-m gpu``; skipped with fewer than two H100s).

The kernels that take more than 48 KB of dynamic shared memory (the AHC merge kernel, the fused VBx E-step and the
fused centroid accumulation) must be opted in on every device they run on: a function attribute holds for the device
that was current when it was set.  Each pooled call context sets them on its own device when it is made (the pool keeps
one context per device and concurrent caller), so a call on device 1 after one on device 0 runs the same kernels and
gives the same labels.
"""
import numpy as np
import pytest

from fluidaudio_b200 import _lib, synth
from fluidaudio_b200.clustering import OfflineClusterer

pytestmark = pytest.mark.gpu


def test_diarize_cluster_on_device_1_after_device_0(gpu_lib):
    if _lib.device_count() < 2:
        pytest.skip("needs two sm_90a devices")
    # 5 000 rows: the merge kernel keeps its master state in shared memory; four speakers: fused VBx and centroids
    emb, _ = synth.speaker_embeddings(5000, 256, 4, seed=21)
    rho, psi = synth.synthetic_plda(emb)
    results = []
    try:
        for dev in (0, 1):
            _lib.set_device(dev)
            results.append(OfflineClusterer(psi=psi).cluster(emb, rho))
    finally:
        _lib.set_device(0)
    a, b = results
    assert a.info["initial_clusters"] <= 64 and a.info["training_count"] == 5000
    assert np.array_equal(a.labels, b.labels)
    assert np.array_equal(a.centroids, b.centroids)
