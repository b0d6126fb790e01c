"""Offline Sortformer diarization on the GPU (``include/fluidaudio_b200_offline_sortformer.h``): what
OfflineSortformerDiarizer.processComplete (Sources/FluidAudio/Diarizer/Sortformer/Offline/) does between the log-mel
and the timeline, for every window of many files per launch.  The fused ``mel -> speaker_preds`` model stays with the
caller.

* ``OfflineSortformerConfig``: the fixed window geometry and the one knob, ``overlap_output_frames``.
* ``OfflineSortformerWindows``: ``plan``, ``model_inputs`` (every window's channels-first mel and mel_length) and
  ``stitch`` (the windows' speaker columns aligned and averaged into one row set per file), each with host arrays or,
  in the ``*_device`` form, raw HBM pointers.
* ``OfflineSortformerDiarizer.process_complete_batch``: the whole pipeline, from samples to one finalized
  ``DiarizerTimeline`` per clip.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence

import numpy as np

from . import _lib
from .diarizer_timeline import SEGMENT, DiarizerTimeline, DiarizerTimelineConfig, DiarizerTimelines

WINDOW_OUT = 384      # FA_OFFLINE_SORTFORMER_WINDOW_OUT
SUBSAMPLING = 8       # FA_OFFLINE_SORTFORMER_SUBSAMPLING
WINDOW_MEL = 3072     # FA_OFFLINE_SORTFORMER_WINDOW_MEL
SPEAKERS = 4          # FA_OFFLINE_SORTFORMER_SPEAKERS
MELS = 128            # FA_OFFLINE_SORTFORMER_MELS
WINDOW_BYTES = MELS * WINDOW_MEL * 4   # one window's model input, 1.5 MB


@dataclass
class OfflineSortformerConfig:
    """OfflineSortformerConfig (OfflineSortformerDiarizer.swift:13-58) without the model precision, which selects the
    caller's model."""
    overlap_output_frames: int = 100
    window_output_frames: int = field(default=WINDOW_OUT, init=False)
    subsampling_factor: int = field(default=SUBSAMPLING, init=False)
    num_speakers: int = field(default=SPEAKERS, init=False)
    mel_features: int = field(default=MELS, init=False)
    sample_rate: int = field(default=16000, init=False)
    mel_window: int = field(default=400, init=False)
    mel_stride: int = field(default=160, init=False)

    @classmethod
    def offline_v2_1(cls) -> "OfflineSortformerConfig":
        return cls()

    @property
    def window_mel_frames(self) -> int:
        return self.window_output_frames * self.subsampling_factor

    @property
    def frame_duration_seconds(self) -> float:
        """Float(subsamplingFactor) * Float(melStride) / Float(sampleRate), in float32"""
        f = np.float32
        return float(f(f(self.subsampling_factor) * f(self.mel_stride)) / f(self.sample_rate))


class OfflineSortformerWindows:
    """The fa_offline_sortformer_* calls on the current device"""

    def __init__(self):
        self._L = _lib.load()

    def plan(self, mel_frames, overlap: int = 100):
        """(window_counts, output_frames) int64 per file"""
        n = np.ascontiguousarray(mel_frames, np.int64).reshape(-1)
        w, r = np.zeros(n.size, np.int64), np.zeros(n.size, np.int64)
        _lib.check(self._L.fa_offline_sortformer_plan(int(overlap), n.size, _lib.ptr(n), _lib.ptr(w), _lib.ptr(r)),
                   "fa_offline_sortformer_plan")
        return w, r

    def model_inputs(self, mel, mel_offsets, mel_frames, overlap: int = 100):
        """(mel [W x 128 x 3072], mel_length [W] int32) for the files' time-major rows in ``mel`` (flat float32) at
        ``mel_offsets`` floats"""
        m = np.ascontiguousarray(mel, np.float32).reshape(-1)
        off = np.ascontiguousarray(mel_offsets, np.int64).reshape(-1)
        n = np.ascontiguousarray(mel_frames, np.int64).reshape(-1)
        W = int(self.plan(n, overlap)[0].sum())
        out, ml = np.empty((W, MELS, WINDOW_MEL), np.float32), np.empty(W, np.int32)
        _lib.check(self._L.fa_offline_sortformer_model_inputs(int(overlap), n.size, _lib.ptr(m) if m.size else None,
                                                              _lib.ptr(off), _lib.ptr(n), W, _lib.ptr(out),
                                                              _lib.ptr(ml)), "fa_offline_sortformer_model_inputs")
        return out, ml

    def model_inputs_device(self, d_mel, mel_offsets, mel_frames, window_capacity, d_model_mel, d_mel_length,
                            overlap: int = 100):
        off = np.ascontiguousarray(mel_offsets, np.int64).reshape(-1)
        n = np.ascontiguousarray(mel_frames, np.int64).reshape(-1)
        _lib.check(self._L.fa_offline_sortformer_model_inputs_device(int(overlap), n.size, d_mel, _lib.ptr(off),
                                                                     _lib.ptr(n), int(window_capacity), d_model_mel,
                                                                     d_mel_length),
                   "fa_offline_sortformer_model_inputs_device")

    def stitch(self, speaker_preds, mel_frames, overlap: int = 100, mappings: bool = False):
        """predictions [sum of output_frames x 4] packed in file order (and, with ``mappings``, [W x 4] int32)"""
        n = np.ascontiguousarray(mel_frames, np.int64).reshape(-1)
        w, r = self.plan(n, overlap)
        p = np.ascontiguousarray(speaker_preds, np.float32).reshape(-1)
        assert p.size == int(w.sum()) * WINDOW_OUT * SPEAKERS, "speaker_preds does not hold [windows x 384 x 4]"
        out = np.empty((int(r.sum()), SPEAKERS), np.float32)
        maps = np.empty((int(w.sum()), SPEAKERS), np.int32) if mappings else None
        _lib.check(self._L.fa_offline_sortformer_stitch(int(overlap), n.size, _lib.ptr(n), _lib.ptr(p) if p.size else
                                                        None, _lib.ptr(out) if out.size else None, _lib.ptr(maps)),
                   "fa_offline_sortformer_stitch")
        return (out, maps) if mappings else out

    def stitch_device(self, d_speaker_preds, mel_frames, d_predictions, d_mappings=None, overlap: int = 100):
        n = np.ascontiguousarray(mel_frames, np.int64).reshape(-1)
        _lib.check(self._L.fa_offline_sortformer_stitch_device(int(overlap), n.size, _lib.ptr(n), d_speaker_preds,
                                                               d_predictions, d_mappings),
                   "fa_offline_sortformer_stitch_device")


class OfflineSortformerDiarizer:
    """OfflineSortformerDiarizer over a caller model:
      model(mel [B x 128 x 3072] float32, mel_length [B] int32) -> speaker_preds [B x 384 x 4] float32
    (numpy in, numpy out).  Each call's windows go to the model in groups of at most ``window_budget`` windows
    (1.5 MB of model input each); a file's windows are never split across groups, so a file longer than the budget
    forms a group of its own."""

    def __init__(self, model: Callable, config: Optional[OfflineSortformerConfig] = None,
                 timeline_config: Optional[DiarizerTimelineConfig] = None, window_budget: int = 256):
        from .mel import AudioMelSpectrogram
        self.model = model
        self.config = config or OfflineSortformerConfig.offline_v2_1()
        self.timeline_config = timeline_config or DiarizerTimelineConfig.default(self.config.num_speakers,
                                                                                 self.config.frame_duration_seconds)
        self.window_budget = max(1, int(window_budget))
        self.mel = AudioMelSpectrogram()
        self.windows = OfflineSortformerWindows()

    def process_complete(self, samples, source_sample_rate: Optional[float] = None) -> DiarizerTimeline:
        return self.process_complete_batch([samples], source_sample_rate)[0]

    def _normalize(self, samples, source_sample_rate):
        a = np.ascontiguousarray(samples, np.float32).reshape(-1)
        if source_sample_rate is None or float(source_sample_rate) == float(self.config.sample_rate):
            return a
        from .audio_converter import AudioConverter
        return AudioConverter(float(self.config.sample_rate)).resample(a, float(source_sample_rate))

    def _groups(self, windows):
        groups, cur, used = [], [], 0
        for i, w in enumerate(windows.tolist()):
            if cur and used + w > self.window_budget:
                groups.append(cur)
                cur, used = [], 0
            cur.append(i)
            used += w
        if cur:
            groups.append(cur)
        return groups

    def process_complete_batch(self, clips: Sequence, source_sample_rate: Optional[float] = None
                               ) -> List[DiarizerTimeline]:
        """processComplete for every clip: one finalized DiarizerTimeline each (an empty clip gets a fresh one)."""
        ov = int(self.config.overlap_output_frames)
        audio = [self._normalize(c, source_sample_rate) for c in clips]
        live = [i for i, a in enumerate(audio) if a.size > 0]
        rows = np.zeros(len(audio), np.int64)
        if live:
            # the log-mel of every clip in one call, kept in HBM
            offsets = np.concatenate([[0], np.cumsum([audio[i].size for i in live])]).astype(np.int64)
            out_offsets = np.zeros(len(live) + 1, np.int64)
            for j, i in enumerate(live):
                out_offsets[j + 1] = out_offsets[j] + max(self.mel.frame_count(audio[i].size), 1) * MELS
            d_audio = _lib.DeviceBuffer(int(offsets[-1]) * 4)
            d_audio.upload(np.concatenate([audio[i] for i in live]))
            d_mel = _lib.DeviceBuffer(int(out_offsets[-1]) * 4)
            _, nf = self.mel.compute_batch_device(d_audio, offsets, d_mel, out_offsets)
            d_audio.free()
            wins, outs = self.windows.plan(nf, ov)
            rows[live] = outs
            # every file's stitched rows, packed in file order: the finalized rows of one timeline push
            d_rows = _lib.DeviceBuffer(max(int(outs.sum()), 1) * SPEAKERS * 4)
            row_at = np.concatenate([[0], np.cumsum(outs)])
            for group in self._groups(wins):
                self._run_group(group, d_mel, out_offsets, nf, wins, d_rows, int(row_at[group[0]]), ov)
            d_mel.free()
        cfg = DiarizerTimelineConfig(**{k: getattr(self.timeline_config, k) for k in
                                        DiarizerTimelineConfig.__dataclass_fields__})
        cfg.max_stored_frames = max(1, int(rows.max()) if rows.size else 1)   # the reference keeps every row
        tls = DiarizerTimelines(cfg, max_tentative_rows=0)
        timelines = [tls.open() for _ in audio]
        if live:
            self._rebuild(tls, [timelines[i] for i in live], d_rows, outs)
        return timelines

    def _run_group(self, group, d_mel, out_offsets, nf, wins, d_rows, row0, ov):
        """model inputs, the model and the stitch for the files ``group`` (indices into the live files)"""
        W = int(wins[group].sum())
        if W == 0:
            return
        d_in = _lib.DeviceBuffer(W * WINDOW_BYTES)
        d_len = _lib.DeviceBuffer(W * 4)
        self.windows.model_inputs_device(d_mel.ptr, out_offsets[group], nf[group], W, d_in.ptr, d_len.ptr, ov)
        _lib.synchronize()
        mel = d_in.download((W, MELS, WINDOW_MEL), np.float32)
        mel_length = d_len.download(W, np.int32)
        d_in.free()
        sp = np.ascontiguousarray(self.model(mel, mel_length), np.float32).reshape(W, WINDOW_OUT, SPEAKERS)
        d_sp = _lib.DeviceBuffer(sp.nbytes)
        d_sp.upload(sp)
        self.windows.stitch_device(d_sp.ptr, nf[group], d_rows.ptr.value + row0 * SPEAKERS * 4, None, ov)
        _lib.synchronize()
        d_sp.free()

    @staticmethod
    def _rebuild(tls, timelines, d_rows, rows):
        """rebuild(finalizedPredictions:tentativePredictions: [], keepingSpeakers: false, isComplete: true) of fresh
        sessions: one push of every file's rows, then finalize"""
        n = len(timelines)
        ten = np.zeros(n, np.int64)
        bf, bt = tls.segment_bound(rows, ten)
        d_fs, d_ts = _lib.DeviceBuffer(max(bf, 1) * SEGMENT.itemsize), _lib.DeviceBuffer(max(bt, 1) * SEGMENT.itemsize)
        d_fc, d_tc = _lib.DeviceBuffer(n * 8), _lib.DeviceBuffer(n * 8)
        ids = [t.session for t in timelines]
        tls.push_device(ids, d_rows, rows, d_rows, ten, d_fs, d_ts, d_fc, d_tc)
        _lib.synchronize()
        fc, tc = d_fc.download(n, np.int64), d_tc.download(n, np.int64)
        fs = d_fs.download(int(fc.sum()), SEGMENT)
        ts = d_ts.download(int(tc.sum()), SEGMENT)
        tls.finalize(ids)
        fo, to = np.concatenate([[0], np.cumsum(fc)]), np.concatenate([[0], np.cumsum(tc)])
        for j, t in enumerate(timelines):
            t._apply(fs[fo[j]:fo[j + 1]], ts[to[j]:to[j + 1]])
            for sp in t.speakers.values():
                sp.finalize()
