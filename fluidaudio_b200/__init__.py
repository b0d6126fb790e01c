"""fluidaudio_b200 — H100-native (sm_90a) implementation of FluidAudio's two CPU hot paths.

* log-mel frontend:  :class:`fluidaudio_b200.mel.AudioMelSpectrogram`
* offline clustering backend:  :class:`fluidaudio_b200.clustering.AHCClustering`, ``VBxClustering``,
  ``OfflineClusterer`` and the drop-in C symbol ``fastcluster_compute_centroid_linkage``
* offline diarization's prepare stage:  :class:`fluidaudio_b200.segmentation.OfflineSegmentationProcessor`,
  ``OfflineEmbeddingPlanner``, ``WeightInterpolation``

The compute lives in ``lib/libfluidaudio_b200.so`` (CUDA, C ABI in ``include/``).  Importing this package does not
load it; the first call does, and raises if the library is missing or no H100 is visible (no CPU fallback).
"""
from ._lib import FluidAudioError, device_count, kernel_launch_count, set_device, synchronize  # noqa: F401

__all__ = ["FluidAudioError", "device_count", "kernel_launch_count", "set_device", "synchronize"]
