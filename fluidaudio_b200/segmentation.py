"""Host-side mirror of the offline diarizer's prepare stage: what ``OfflineDiarizerManager.prepare`` computes around the
segmentation and embedding networks (which run outside this library, e.g. in PyTorch on the same GPU).

* :class:`OfflineSegmentationProcessor` — Diarizer/Offline/Segmentation/OfflineSegmentationProcessor.swift: analysis
  windows (:55-56, 118-190), powerset decoding into ``SegmentationOutput`` (:321-405, 527-535).
* :class:`OfflineEmbeddingPlanner` — Diarizer/Offline/Extraction/OfflineEmbeddingExtractor.swift:421-707: which (chunk,
  local speaker) pairs get an embedding, their masks, the weights the embedding network takes, the fbank windows and the
  ``TimedEmbedding`` metadata that ``cluster(_:)`` and the export file need.
* :class:`WeightInterpolation` — Diarizer/Offline/Extraction/WeightInterpolation.swift.

All arithmetic happens in the sm_90a kernels behind ``fa_seg_*`` / ``fa_embedding_plan`` / ``fa_embed_windows`` /
``fa_weight_resample``.  The ``*_device`` methods take :class:`fluidaudio_b200._lib.DeviceBuffer` objects (or anything
with a ``ptr`` attribute holding a device address) for the large buffers and leave their results on the device.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _lib
from .export_io import EmbeddingExport, PreparedDiarization

COUNTER_NAMES = ("evaluated", "empty", "fallback", "skipped")


@dataclass
class SegmentationConfig:             # OfflineDiarizerConfig.Segmentation.community
    sample_rate: int = 16000
    window_duration: float = 10.0
    step_ratio: float = 0.2
    speech_onset_threshold: float = 0.5

    def _c(self) -> _lib.SegConfig:
        return _lib.SegConfig(self.sample_rate, self.speech_onset_threshold, self.window_duration, self.step_ratio)


@dataclass
class EmbeddingPlanConfig:            # OfflineDiarizerConfig.Embedding.community + the embedding network's shapes
    exclude_overlap: bool = True
    min_segment_duration: float = 1.0
    skip_threshold: float | None = None    # EmbeddingSkipStrategy.maskSimilarity(threshold); None = .none
    weight_frames: int = 589
    audio_sample_count: int = 160000
    fbank_batch: int = 32                  # min(modelBatchLimit, 32)

    def _c(self) -> _lib.EmbedPlanConfig:
        return _lib.EmbedPlanConfig(int(self.exclude_overlap), -1.0 if self.skip_threshold is None else self.skip_threshold,
                                    self.min_segment_duration, self.weight_frames, self.audio_sample_count,
                                    self.fbank_batch, 0)


@dataclass
class SegmentationOutput:             # OfflineDiarizerTypes.swift SegmentationOutput, plus the two tallies of the decoder
    log_probs: np.ndarray             # float32 [numChunks, numFrames, classes]
    speaker_weights: np.ndarray       # float32 [numChunks, numFrames, numSpeakers]
    num_chunks: int
    num_frames: int
    num_speakers: int
    chunk_offsets: np.ndarray         # float64 [numChunks]
    frame_duration: float
    class_histogram: np.ndarray = field(default_factory=lambda: np.zeros(8, np.int64))
    speech_frames: int = 0


def _dptr(buf):
    return None if buf is None else buf.ptr


class OfflineSegmentationProcessor:
    def __init__(self, config: SegmentationConfig | None = None):
        self.config = config or SegmentationConfig()

    def window_count(self, total_samples: int) -> tuple[int, int, int]:
        """(windows, samplesPerWindow, samplesPerStep) for an audio of `total_samples` samples; host arithmetic."""
        n, w, s = C.c_int32(), C.c_int64(), C.c_int64()
        cfg = self.config._c()
        _lib.check(_lib.load().fa_seg_window_count(int(total_samples), C.byref(cfg), C.byref(n), C.byref(w), C.byref(s)),
                   "fa_seg_window_count")
        return n.value, w.value, s.value

    def windows(self, audio, first_chunk: int = 0, chunk_count: int | None = None) -> tuple[np.ndarray, np.ndarray]:
        """(windows float32 [count, samplesPerWindow], chunkOffsets float64 [count]); an empty audio raises, as the
        reference throws noSpeechDetected."""
        a = np.ascontiguousarray(audio, np.float32).reshape(-1)
        n, w, _ = self.window_count(a.size)
        count = n - first_chunk if chunk_count is None else chunk_count
        out, offs = np.zeros((max(count, 0), w), np.float32), np.zeros(max(count, 0), np.float64)
        cfg = self.config._c()
        _lib.check(_lib.load().fa_seg_windows(_lib.ptr(a) if a.size else None, a.size, C.byref(cfg), first_chunk, count,
                                              _lib.ptr(out), _lib.ptr(offs)), "fa_seg_windows")
        return out, offs

    def windows_device(self, d_audio, total_samples: int, d_out, first_chunk: int, chunk_count: int) -> np.ndarray:
        """Windows gathered from a device audio buffer into d_out [chunk_count x samplesPerWindow]; returns the offsets."""
        offs = np.zeros(chunk_count, np.float64)
        cfg = self.config._c()
        _lib.check(_lib.load().fa_seg_windows_device(_dptr(d_audio), int(total_samples), C.byref(cfg), first_chunk,
                                                     chunk_count, _dptr(d_out), _lib.ptr(offs)), "fa_seg_windows_device")
        return offs

    def decode(self, logits, chunk_offsets=None, want_log_probs: bool = True) -> SegmentationOutput:
        """logits [chunks, frames, classes] (the segmentation network's output for the windows in order)."""
        x = np.ascontiguousarray(logits, np.float32)
        if x.ndim == 2:
            x = x[None]
        c, f, k = x.shape
        lp = np.zeros((c, f, k), np.float32) if want_log_probs else None
        w = np.zeros((c, f, 3), np.float32)
        hist, speech = np.zeros(8, np.int64), C.c_int64()
        cfg = self.config._c()
        _lib.check(_lib.load().fa_seg_decode(_lib.ptr(x) if x.size else None, c, f, k, C.byref(cfg), _lib.ptr(lp),
                                             _lib.ptr(w) if w.size else None, hist.ctypes.data, C.byref(speech)),
                   "fa_seg_decode")
        if chunk_offsets is None:
            step = self.window_count(1)[2]
            chunk_offsets = np.arange(c, dtype=np.float64) * step / float(self.config.sample_rate)
        return SegmentationOutput(lp if want_log_probs else np.zeros((c, f, k), np.float32), w, c, f, 3,
                                  np.ascontiguousarray(chunk_offsets, np.float64),
                                  self.config.window_duration / f if f else 0.0, hist, speech.value)

    def decode_device(self, d_logits, chunks: int, frames: int, classes: int, d_log_probs, d_speaker_weights):
        """Device buffers in and out (d_log_probs may be None); returns (class_histogram int64 [8], speech_frames)."""
        hist, speech = np.zeros(8, np.int64), C.c_int64()
        cfg = self.config._c()
        _lib.check(_lib.load().fa_seg_decode_device(_dptr(d_logits), chunks, frames, classes, C.byref(cfg),
                                                    _dptr(d_log_probs), _dptr(d_speaker_weights), hist.ctypes.data,
                                                    C.byref(speech)), "fa_seg_decode_device")
        return hist, speech.value


@dataclass
class EmbeddingPlan:
    """One row per embedding the reference would extract, in its order (chunk-major, speaker-minor)."""
    chunk_index: np.ndarray           # int32 [M]   TimedEmbedding.chunkIndex
    speaker_index: np.ndarray         # int32 [M]   .speakerIndex
    start_frame: np.ndarray           # int32 [M]   .startFrame
    end_frame: np.ndarray             # int32 [M]   .endFrame
    start_time: np.ndarray            # float64 [M] .startTime
    end_time: np.ndarray              # float64 [M] .endTime
    mask_sum: np.ndarray              # float32 [M]
    used_fallback: np.ndarray         # int32 [M]   the base mask replaced a too short clean mask
    reuse_of: np.ndarray              # int32 [M]   entry whose embedding the skip strategy reuses, -1 = its own
    frame_weights: np.ndarray         # float32 [M, frames]         .frameWeights
    model_weights: np.ndarray         # float32 [M, weight_frames]  the embedding network's weights input
    counters: dict                    # evaluated, empty, fallback, skipped
    num_chunks: int = 0
    num_speakers: int = 0

    @property
    def count(self) -> int:
        return int(self.chunk_index.size)

    def expand_embeddings(self, computed: np.ndarray) -> np.ndarray:
        """Rows for every entry from the rows of the entries that ran the embedding network (reuse_of < 0), in order."""
        own = np.flatnonzero(self.reuse_of < 0)
        computed = np.asarray(computed)
        assert computed.shape[0] == own.size, (computed.shape, own.size)
        where = np.full(self.count, -1, np.int64)
        where[own] = np.arange(own.size)
        src = np.where(self.reuse_of < 0, where, where[np.maximum(self.reuse_of, 0)])
        return computed[src]

    def to_prepared(self, embedding256, rho128) -> PreparedDiarization:
        """The input of ``export_io.cluster_prepared`` and the export file, from this plan's metadata and the networks'
        outputs for its entries."""
        emb = np.ascontiguousarray(embedding256, np.float32)
        rho = np.ascontiguousarray(rho128, np.float64)
        assert emb.shape[0] == self.count and rho.shape[0] == self.count
        export = EmbeddingExport(self.chunk_index, self.speaker_index, self.start_frame, self.end_frame, self.start_time,
                                 self.end_time, emb, rho, np.full(self.count, -1, np.int32))
        return PreparedDiarization(export, self.num_chunks, self.num_speakers, {})


class OfflineEmbeddingPlanner:
    def __init__(self, segmentation: SegmentationConfig | None = None, config: EmbeddingPlanConfig | None = None):
        self.segmentation = segmentation or SegmentationConfig()
        self.config = config or EmbeddingPlanConfig()

    def plan(self, segmentation: SegmentationOutput, total_samples: int) -> EmbeddingPlan:
        w = np.ascontiguousarray(segmentation.speaker_weights, np.float32)
        c, f, s = w.shape if w.ndim == 3 else (0, 0, 0)
        offs = np.ascontiguousarray(segmentation.chunk_offsets, np.float64)
        cap, wf = max(c * s, 1), self.config.weight_frames
        i32 = lambda: np.zeros(cap, np.int32)
        ci, si, sf, ef, fb, ro = i32(), i32(), i32(), i32(), i32(), i32()
        st, et, ms = np.zeros(cap, np.float64), np.zeros(cap, np.float64), np.zeros(cap, np.float32)
        fw, mw = np.zeros((cap, max(f, 1)), np.float32), np.zeros((cap, wf), np.float32)
        n, counters = C.c_int32(), np.zeros(4, np.int64)
        seg, cfg = self.segmentation._c(), self.config._c()
        _lib.check(_lib.load().fa_embedding_plan(
            _lib.ptr(w) if w.size else None, c, f, s, _lib.ptr(offs) if offs.size else None, offs.size,
            float(segmentation.frame_duration), int(total_samples), C.byref(seg), C.byref(cfg), _lib.ptr(ci), _lib.ptr(si),
            _lib.ptr(sf), _lib.ptr(ef), _lib.ptr(st), _lib.ptr(et), _lib.ptr(ms), _lib.ptr(fb), _lib.ptr(ro), _lib.ptr(fw),
            _lib.ptr(mw), C.byref(n), counters.ctypes.data), "fa_embedding_plan")
        m = n.value
        return EmbeddingPlan(ci[:m], si[:m], sf[:m], ef[:m], st[:m], et[:m], ms[:m], fb[:m], ro[:m], fw[:m, :f], mw[:m],
                             dict(zip(COUNTER_NAMES, counters.tolist())), c, s)

    def plan_device(self, d_speaker_weights, chunks: int, frames: int, speakers: int, chunk_offsets,
                    frame_duration: float, total_samples: int, d_out: dict) -> tuple[int, dict]:
        """Device weights in, per-entry device arrays out.  `d_out` maps any of chunk_index, speaker_index, start_frame,
        end_frame, start_time, end_time, mask_sum, used_fallback, reuse_of, frame_weights, model_weights to a device
        buffer of capacity chunks * speakers entries; returns (entry count, counters)."""
        names = ("chunk_index", "speaker_index", "start_frame", "end_frame", "start_time", "end_time", "mask_sum",
                 "used_fallback", "reuse_of", "frame_weights", "model_weights")
        unknown = set(d_out) - set(names)
        if unknown:
            raise ValueError(f"unknown outputs: {sorted(unknown)}")
        offs = np.ascontiguousarray(chunk_offsets if chunk_offsets is not None else [], np.float64)
        n, counters = C.c_int32(), np.zeros(4, np.int64)
        seg, cfg = self.segmentation._c(), self.config._c()
        _lib.check(_lib.load().fa_embedding_plan_device(
            _dptr(d_speaker_weights), chunks, frames, speakers, _lib.ptr(offs) if offs.size else None, offs.size,
            float(frame_duration), int(total_samples), C.byref(seg), C.byref(cfg), *[_dptr(d_out.get(k)) for k in names],
            C.byref(n), counters.ctypes.data), "fa_embedding_plan_device")
        return n.value, dict(zip(COUNTER_NAMES, counters.tolist()))

    def fbank_windows(self, audio, chunk_offsets, chunk_index=None, count: int | None = None) -> np.ndarray:
        """The fbank input rows [count, audio_sample_count] of the listed chunks (all of chunk_offsets by default)."""
        a = np.ascontiguousarray(audio, np.float32).reshape(-1)
        offs = np.ascontiguousarray(chunk_offsets if chunk_offsets is not None else [], np.float64)
        idx = None if chunk_index is None else np.ascontiguousarray(chunk_index, np.int32)
        count = (offs.size if idx is None else idx.size) if count is None else count
        out = np.zeros((count, self.config.audio_sample_count), np.float32)
        seg = self.segmentation._c()
        _lib.check(_lib.load().fa_embed_windows(_lib.ptr(a) if a.size else None, a.size, _lib.ptr(offs) if offs.size else None,
                                                offs.size, _lib.ptr(idx), count, C.byref(seg),
                                                self.config.audio_sample_count, _lib.ptr(out) if out.size else None),
                   "fa_embed_windows")
        return out

    def fbank_windows_device(self, d_audio, total_samples: int, chunk_offsets, chunk_index, count: int, d_out) -> None:
        offs = np.ascontiguousarray(chunk_offsets if chunk_offsets is not None else [], np.float64)
        idx = None if chunk_index is None else np.ascontiguousarray(chunk_index, np.int32)
        seg = self.segmentation._c()
        _lib.check(_lib.load().fa_embed_windows_device(_dptr(d_audio), int(total_samples),
                                                       _lib.ptr(offs) if offs.size else None, offs.size, _lib.ptr(idx),
                                                       count, C.byref(seg), self.config.audio_sample_count, _dptr(d_out)),
                   "fa_embed_windows_device")


class WeightInterpolation:
    """WeightInterpolation.swift: half-pixel linear interpolation in float32 (scipy.ndimage.zoom(order=1) mapping)."""

    @staticmethod
    def resample_2d(rows, output_length: int) -> np.ndarray:
        r = np.ascontiguousarray(rows, np.float32)
        if r.ndim != 2 or r.shape[0] == 0 or r.shape[1] == 0 or output_length <= 0:
            return np.zeros((0, 0), np.float32)
        out = np.zeros((r.shape[0], output_length), np.float32)
        _lib.check(_lib.load().fa_weight_resample(_lib.ptr(r), r.shape[0], r.shape[1], output_length, _lib.ptr(out)),
                   "fa_weight_resample")
        return out

    @staticmethod
    def resample(values, output_length: int) -> np.ndarray:
        v = np.ascontiguousarray(values, np.float32).reshape(-1)
        if v.size == 0 or output_length <= 0:
            return np.zeros(0, np.float32)
        return WeightInterpolation.resample_2d(v[None], output_length)[0]

    @staticmethod
    def zoom(values, factor: float) -> np.ndarray:
        v = np.ascontiguousarray(values, np.float32).reshape(-1)
        if v.size == 0 or not factor > 0:
            return np.zeros(0, np.float32)
        scaled = float(np.float32(v.size) * np.float32(factor))
        rounded = np.floor(abs(scaled) + 0.5) * (1 if scaled >= 0 else -1)   # Float.rounded(): ties away from zero
        return WeightInterpolation.resample(v, max(1, int(rounded)))
