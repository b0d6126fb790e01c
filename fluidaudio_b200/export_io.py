"""Embedding-export files and the cacheable clustering input (SURVEY.md 8f rank 2).

Reference: OfflineDiarizerManager.exportEmbeddings (Sources/FluidAudio/Diarizer/Offline/Core/OfflineDiarizerManager.swift:913-955)
writes `[TimedEmbedding + cluster]` as JSON when `OfflineDiarizerConfig.embeddingExportPath` is set; `PreparedDiarization`
(PreparedDiarization.swift:8-26) is the in-memory cache that `OfflineDiarizerManager.cluster(_:)` consumes so that
clustering can be re-run without model inference.  Here the file is the wire format between a Mac running the CoreML
models and the GPU clustering backend: parsing is native (`fa_export_*` in libfluidaudio_b200.so).
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field

import numpy as np

from . import _lib
from .clustering import ClusterResult, OfflineClusterer, OfflineDiarizerConfig, build_chunk_assignments


@dataclass
class EmbeddingExport:
    """Column-wise view of an export file: entry i is TimedEmbedding i (OfflineDiarizerTypes.swift:706-716) plus the
    cluster id the writer assigned (-1 when it had none)."""
    chunk_index: np.ndarray      # int32 [N]
    speaker_index: np.ndarray    # int32 [N]
    start_frame: np.ndarray      # int32 [N]
    end_frame: np.ndarray        # int32 [N]
    start_time: np.ndarray       # float64 [N]
    end_time: np.ndarray         # float64 [N]
    embedding256: np.ndarray     # float32 [N, E]
    rho128: np.ndarray           # float64 [N, R]
    cluster: np.ndarray          # int32 [N]

    @property
    def count(self) -> int:
        return int(self.embedding256.shape[0])

    @staticmethod
    def read(path: str | os.PathLike) -> "EmbeddingExport":
        L = _lib.load()
        p = os.fsencode(path)
        n, e, r = C.c_size_t(), C.c_size_t(), C.c_size_t()
        _lib.check(L.fa_export_shape(p, C.byref(n), C.byref(e), C.byref(r)), "fa_export_shape")
        N, E, R = n.value, e.value, r.value
        out = EmbeddingExport(np.zeros(N, np.int32), np.zeros(N, np.int32), np.zeros(N, np.int32), np.zeros(N, np.int32),
                              np.zeros(N, np.float64), np.zeros(N, np.float64), np.zeros((N, E), np.float32),
                              np.zeros((N, R), np.float64), np.zeros(N, np.int32))
        if N:
            _lib.check(L.fa_export_read(p, N, E, R, out.chunk_index.ctypes.data, out.speaker_index.ctypes.data,
                                        out.start_frame.ctypes.data, out.end_frame.ctypes.data,
                                        out.start_time.ctypes.data, out.end_time.ctypes.data,
                                        out.embedding256.ctypes.data, out.rho128.ctypes.data, out.cluster.ctypes.data),
                       "fa_export_read")
        return out

    def write(self, path: str | os.PathLike) -> None:
        a = lambda x, t: np.ascontiguousarray(x, t)
        ci, si = a(self.chunk_index, np.int32), a(self.speaker_index, np.int32)
        sf, ef = a(self.start_frame, np.int32), a(self.end_frame, np.int32)
        st, et = a(self.start_time, np.float64), a(self.end_time, np.float64)
        emb, rho, cl = a(self.embedding256, np.float32), a(self.rho128, np.float64), a(self.cluster, np.int32)
        N = emb.shape[0]
        _lib.check(_lib.load().fa_export_write(os.fsencode(path), N, emb.shape[1] if emb.ndim == 2 else 0,
                                               rho.shape[1] if rho.ndim == 2 else 0, ci.ctypes.data, si.ctypes.data,
                                               sf.ctypes.data, ef.ctypes.data, st.ctypes.data, et.ctypes.data,
                                               emb.ctypes.data, rho.ctypes.data, cl.ctypes.data), "fa_export_write")


@dataclass
class PreparedDiarization:
    """What `cluster(_:)` needs from the (not re-implemented) segmentation + embedding stages, kept so that clustering
    can be repeated with other settings.  Mirrors PreparedDiarization.swift: `embedding_count`,
    `segmentation_chunk_count`; the audio source and segmentation logits stay on the Mac."""
    export: EmbeddingExport
    num_chunks: int = 0
    num_local_speakers: int = 0
    timings: dict = field(default_factory=dict)

    @staticmethod
    def from_export(export: EmbeddingExport) -> "PreparedDiarization":
        nc = int(export.chunk_index.max()) + 1 if export.count else 0
        ns = int(export.speaker_index.max()) + 1 if export.count else 0
        return PreparedDiarization(export, nc, ns)

    @staticmethod
    def load(path) -> "PreparedDiarization":
        return PreparedDiarization.from_export(EmbeddingExport.read(path))

    @property
    def embedding_count(self) -> int:
        return self.export.count

    @property
    def segmentation_chunk_count(self) -> int:
        return self.num_chunks


@dataclass
class ReplayResult:
    result: ClusterResult
    chunk_assignments: np.ndarray        # [num_chunks, num_local_speakers], -2 = inactive (buildChunkAssignments)
    matches_export: bool | None          # same partition as the file's `cluster` column (None: file had no labels)


def cluster_prepared(prepared: PreparedDiarization, psi: np.ndarray, config: OfflineDiarizerConfig | None = None,
                     constrained: bool = True) -> ReplayResult:
    """OfflineDiarizerManager.cluster(_:) from the clustering phase on (OfflineDiarizerManager.swift:270-384): AHC ->
    VBx -> centroids -> (constrained) assignment -> per-chunk assignment matrix.  `constrained` follows the
    reference's default `constrainedAssignment: true`."""
    ex = prepared.export
    clusterer = OfflineClusterer(config, psi=psi)
    res = clusterer.cluster(ex.embedding256, ex.rho128, chunk_indices=ex.chunk_index if constrained else None)
    k = int(res.labels.max()) + 1 if ex.count and res.labels.max() >= 0 else 0
    matrix = build_chunk_assignments(ex.chunk_index, ex.speaker_index, res.labels, prepared.num_chunks,
                                     prepared.num_local_speakers, max(k, 1)) if ex.count else np.zeros((0, 0), np.int32)
    same = None
    if ex.count and (ex.cluster >= 0).any():
        same = same_partition(res.labels, ex.cluster)
    return ReplayResult(res, matrix, same)


def same_partition(a, b) -> bool:
    """True when two label vectors describe the same grouping up to a renaming of the ids (entries negative in
    either vector must be negative in both)."""
    a = np.asarray(a).ravel()
    b = np.asarray(b).ravel()
    if a.shape != b.shape:
        return False
    neg_a, neg_b = a < 0, b < 0
    if not np.array_equal(neg_a, neg_b):
        return False
    fwd, back = {}, {}
    for x, y in zip(a[~neg_a].tolist(), b[~neg_b].tolist()):
        if fwd.setdefault(x, y) != y or back.setdefault(y, x) != x:
            return False
    return True
