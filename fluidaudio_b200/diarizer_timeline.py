"""Diarizer timelines on the GPU (``fa_diarizer_timeline_*``): DiarizerTimeline (Diarizer/DiarizerTimeline.swift) for
many live sessions, turning frame-wise speaker probabilities from Sortformer, LS-EEND or any frame-based diarizer into
speech segments.

``DiarizerTimelines`` owns the sessions in HBM; one ``push`` advances every session of a tick.  ``DiarizerTimeline`` is
one session seen as the reference's class: ``add_chunk``, ``finalize``, ``reset``, ``rebuild``, the speakers and their
stored segments (kept here on the host, as the reference keeps them in DiarizerSpeaker) and the probability queries.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field, fields
from types import SimpleNamespace

import numpy as np

from . import _lib

SIGMOIDS, LOGITS = 0, 1
SEGMENT = _lib.TIMELINE_SEGMENT
_C_FIELDS = ("num_speakers", "frame_duration_seconds", "onset_threshold", "offset_threshold", "onset_pad_frames",
             "offset_pad_frames", "min_frames_on", "min_frames_off", "activity_type", "max_stored_frames")


@dataclass
class DiarizerTimelineConfig:
    """DiarizerTimelineConfig (DiarizerTimeline.swift:9-164).  ``max_stored_frames`` caps the finalized predictions kept
    per session (the reference's nil, unlimited, is not offered); ``store_segments`` is the façade's (host) switch."""
    num_speakers: int = 1
    frame_duration_seconds: float = 0.08
    onset_threshold: float = 0.5
    offset_threshold: float = 0.5
    onset_pad_frames: int = 0
    offset_pad_frames: int = 0
    min_frames_on: int = 0
    min_frames_off: int = 0
    activity_type: int = SIGMOIDS
    max_stored_frames: int = 7500
    store_segments: bool = True

    @classmethod
    def default(cls, num_speakers: int, frame_duration_seconds: float) -> "DiarizerTimelineConfig":
        """default(numSpeakers:frameDurationSeconds:): thresholds 0.5, no padding or minimum durations, sigmoids"""
        c = _lib.TimelineConfig()
        _lib.check(_lib.load().fa_diarizer_timeline_default_config(C.byref(c), 0, int(num_speakers),
                                                                   float(frame_duration_seconds)),
                   "fa_diarizer_timeline_default_config")
        return cls._from_c(c)

    @classmethod
    def sortformer_default(cls) -> "DiarizerTimelineConfig":
        """sortformerDefault: 4 speakers, 0.08 s frames"""
        c = _lib.TimelineConfig()
        _lib.check(_lib.load().fa_diarizer_timeline_default_config(C.byref(c), 1, 0, 0.0),
                   "fa_diarizer_timeline_default_config")
        return cls._from_c(c)

    @classmethod
    def from_seconds(cls, onset_pad_seconds: float, offset_pad_seconds: float, min_duration_on: float,
                     min_duration_off: float, **kw) -> "DiarizerTimelineConfig":
        """The seconds initialiser (:139-163): each frame count is Int(round(seconds / frameDurationSeconds)) in
        float32, half away from zero"""
        cfg = cls(**kw)
        c = cfg.to_c()
        _lib.check(_lib.load().fa_diarizer_timeline_config_from_seconds(C.byref(c), onset_pad_seconds,
                                                                        offset_pad_seconds, min_duration_on,
                                                                        min_duration_off),
                   "fa_diarizer_timeline_config_from_seconds")
        out = cls._from_c(c)
        out.store_segments = cfg.store_segments
        return out

    @classmethod
    def _from_c(cls, c) -> "DiarizerTimelineConfig":
        return cls(**{k: getattr(c, k) for k in _C_FIELDS})

    def to_c(self) -> "_lib.TimelineConfig":
        return _lib.TimelineConfig(**{k: getattr(self, k) for k in _C_FIELDS})

    # the seconds accessors (:45-67)
    def _seconds(self, frames: int) -> float:
        return float(np.float32(frames) * np.float32(self.frame_duration_seconds))

    @property
    def onset_pad_seconds(self) -> float:
        return self._seconds(self.onset_pad_frames)

    @property
    def offset_pad_seconds(self) -> float:
        return self._seconds(self.offset_pad_frames)

    @property
    def min_duration_on(self) -> float:
        return self._seconds(self.min_frames_on)

    @property
    def min_duration_off(self) -> float:
        return self._seconds(self.min_frames_off)


@dataclass
class DiarizerSegment:
    """DiarizerSegment (:492-588): frames [start_frame, end_frame) of speaker slot ``speaker_index``."""
    speaker_index: int
    start_frame: int
    end_frame: int
    finalized: bool
    frame_duration_seconds: float
    activity: float = 0.0

    @property
    def length(self) -> int:
        return self.end_frame - self.start_frame

    def _time(self, frames: int) -> float:
        return float(np.float32(frames) * np.float32(self.frame_duration_seconds))

    @property
    def start_time(self) -> float:
        return self._time(self.start_frame)

    @property
    def end_time(self) -> float:
        return self._time(self.end_frame)

    @property
    def duration(self) -> float:
        return self._time(self.end_frame - self.start_frame)


@dataclass
class DiarizerSpeaker:
    """A speaker slot's stored segments (DiarizerSpeaker, :219-487, without enrollment)."""
    index: int
    name: str | None = None
    finalized_segments: list = field(default_factory=list)
    tentative_segments: list = field(default_factory=list)

    def append(self, s: DiarizerSegment):
        (self.finalized_segments if s.finalized else self.tentative_segments).append(s)

    def finalize(self):
        self.finalized_segments.extend(self.tentative_segments)
        self.tentative_segments.clear()

    def reset(self):
        self.finalized_segments.clear()
        self.tentative_segments.clear()


@dataclass
class DiarizerTimelineUpdate:
    finalized_segments: list
    tentative_segments: list


def _ids(sessions):
    return np.ascontiguousarray([int(s) for s in sessions], np.int32)


class DiarizerTimelines:
    """Timeline sessions on the current device.  ``max_tentative_rows`` bounds the tentative rows of one push per
    session.  Not thread-safe, like the reference's timeline."""

    def __init__(self, config: DiarizerTimelineConfig | None = None, max_tentative_rows: int = 64):
        self._L = _lib.load()
        self.config = config or DiarizerTimelineConfig.sortformer_default()
        self.max_tentative_rows = int(max_tentative_rows)
        h = C.c_void_p()
        _lib.check(self._L.fa_diarizer_timeline_create(C.byref(self.config.to_c()), self.max_tentative_rows,
                                                       C.byref(h)), "fa_diarizer_timeline_create")
        self._h = h

    def close_handle(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._L.fa_diarizer_timeline_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close_handle()
        except Exception:
            pass

    # ---- sessions
    def open_session(self) -> int:
        sid = C.c_int32()
        _lib.check(self._L.fa_diarizer_timeline_open(self._h, C.byref(sid)), "fa_diarizer_timeline_open")
        return int(sid.value)

    def open(self) -> "DiarizerTimeline":
        """A fresh session (the lowest free id) as a DiarizerTimeline."""
        return DiarizerTimeline(self, self.open_session())

    def close(self, session):
        sid = session.session if isinstance(session, DiarizerTimeline) else int(session)
        _lib.check(self._L.fa_diarizer_timeline_close(self._h, sid), "fa_diarizer_timeline_close")

    # ---- pushes
    def segment_bound(self, finalized_rows, tentative_rows):
        """(finalized, tentative) segments a push of these per-session row counts may emit"""
        fr, tr = np.ascontiguousarray(finalized_rows, np.int64), np.ascontiguousarray(tentative_rows, np.int64)
        f, t = C.c_int64(), C.c_int64()
        _lib.check(self._L.fa_diarizer_timeline_segment_bound(self.config.num_speakers, fr.size, fr.ctypes.data,
                                                              tr.ctypes.data, C.byref(f), C.byref(t)),
                   "fa_diarizer_timeline_segment_bound")
        return int(f.value), int(t.value)

    def push_packed(self, sessions, finalized, finalized_rows, tentative, tentative_rows):
        """addChunk for every session at once from packed rows ([Σ rows x numSpeakers] each, call order):
        (finalized segments, finalized counts, tentative segments, tentative counts), segments as SEGMENT records."""
        ids = _ids(sessions)
        S = self.config.num_speakers
        fr = np.ascontiguousarray(finalized_rows, np.int64).reshape(-1)
        tr = np.ascontiguousarray(tentative_rows, np.int64).reshape(-1)
        f = np.ascontiguousarray(finalized, np.float32).reshape(-1)
        t = np.ascontiguousarray(tentative, np.float32).reshape(-1)
        assert f.size == fr.sum() * S and t.size == tr.sum() * S, "row counts do not match the packed rows"
        bf, bt = self.segment_bound(fr, tr)
        fo, to = np.zeros(max(bf, 1), SEGMENT), np.zeros(max(bt, 1), SEGMENT)
        fc, tc = np.zeros(ids.size, np.int64), np.zeros(ids.size, np.int64)
        _lib.check(self._L.fa_diarizer_timeline_push(self._h, ids.size, ids.ctypes.data, f.ctypes.data, fr.ctypes.data,
                                                     t.ctypes.data, tr.ctypes.data, fo.ctypes.data, bf, to.ctypes.data,
                                                     bt, fc.ctypes.data, tc.ctypes.data), "fa_diarizer_timeline_push")
        return fo[:fc.sum()], fc, to[:tc.sum()], tc

    def push(self, sessions, finalized, tentative=None):
        """addChunk per session: ``finalized[i]`` / ``tentative[i]`` are [rows x numSpeakers] arrays for sessions[i].
        Returns [(finalized SEGMENT records, tentative SEGMENT records)] per session."""
        S = self.config.num_speakers
        fin = [np.asarray(a, np.float32).reshape(-1, S) for a in finalized]
        ten = [np.zeros((0, S), np.float32)] * len(fin) if tentative is None else \
            [np.asarray(a, np.float32).reshape(-1, S) for a in tentative]
        cat = lambda xs: np.concatenate(xs) if xs else np.zeros((0, S), np.float32)
        fs, fc, ts, tc = self.push_packed(sessions, cat(fin), [a.shape[0] for a in fin], cat(ten),
                                          [a.shape[0] for a in ten])
        fo, to = np.concatenate([[0], np.cumsum(fc)]), np.concatenate([[0], np.cumsum(tc)])
        return [(fs[fo[i]:fo[i + 1]], ts[to[i]:to[i + 1]]) for i in range(len(fin))]

    def push_device(self, sessions, d_finalized: "_lib.DeviceBuffer", finalized_rows, d_tentative: "_lib.DeviceBuffer",
                    tentative_rows, d_finalized_segments: "_lib.DeviceBuffer", d_tentative_segments: "_lib.DeviceBuffer",
                    d_finalized_counts: "_lib.DeviceBuffer", d_tentative_counts: "_lib.DeviceBuffer"):
        """The push on HBM buffers, asynchronous on the handle's stream.  Chains from SortformerStreams.update_device:
        its confirmed / tentative buffers and row counts are ``d_finalized`` / ``finalized_rows`` and ``d_tentative``
        / ``tentative_rows``; call ``_lib.synchronize()`` between the two, since handles do not order each other's
        streams.  Segments (SEGMENT records) and int64 per-session counts go to the four output buffers."""
        ids = _ids(sessions)
        fr = np.ascontiguousarray(finalized_rows, np.int64).reshape(-1)
        tr = np.ascontiguousarray(tentative_rows, np.int64).reshape(-1)
        rec = SEGMENT.itemsize
        _lib.check(self._L.fa_diarizer_timeline_push_device(
            self._h, ids.size, ids.ctypes.data, d_finalized.ptr, fr.ctypes.data, d_tentative.ptr, tr.ctypes.data,
            d_finalized_segments.ptr, d_finalized_segments.nbytes // rec, d_tentative_segments.ptr,
            d_tentative_segments.nbytes // rec, d_finalized_counts.ptr, d_tentative_counts.ptr),
            "fa_diarizer_timeline_push_device")

    def finalize(self, sessions):
        ids = _ids(sessions)
        _lib.check(self._L.fa_diarizer_timeline_finalize(self._h, ids.size, ids.ctypes.data),
                   "fa_diarizer_timeline_finalize")

    def reset(self, sessions):
        ids = _ids(sessions)
        _lib.check(self._L.fa_diarizer_timeline_reset(self._h, ids.size, ids.ctypes.data), "fa_diarizer_timeline_reset")

    def clear_speaker(self, session: int, speaker: int):
        _lib.check(self._L.fa_diarizer_timeline_clear_speaker(self._h, int(session), int(speaker)),
                   "fa_diarizer_timeline_clear_speaker")

    def state(self, session: int):
        """namespace(finalized_frames, stored [rows x S] (oldest first), tentative [rows x S], scratch [S] records)"""
        S = self.config.num_speakers
        info = _lib.TimelineSessionInfo()
        stored = np.zeros((self.config.max_stored_frames, S), np.float32)
        tent = np.zeros((self.max_tentative_rows, S), np.float32)
        scratch = (_lib.TimelineScratch * S)()
        _lib.check(self._L.fa_diarizer_timeline_session_state(self._h, int(session), C.byref(info), stored.ctypes.data,
                                                              tent.ctypes.data, scratch),
                   "fa_diarizer_timeline_session_state")
        sc = np.frombuffer(bytes(scratch), dtype=SCRATCH).copy()
        return SimpleNamespace(finalized_frames=int(info.finalized_frames), stored=stored[:info.stored_frames],
                               tentative=tent[:info.tentative_frames], scratch=sc)

    def add_chunks(self, timelines, finalized, tentative=None):
        """DiarizerTimeline.addChunk for several sessions in one push; returns one DiarizerTimelineUpdate each."""
        raw = self.push([t.session for t in timelines], finalized, tentative)
        return [t._apply(f, g) for t, (f, g) in zip(timelines, raw)]


SCRATCH = np.dtype([(name, np.int64 if t is C.c_int64 else np.float32 if t is C.c_float else np.int32)
                    for name, t in _lib.TimelineScratch._fields_])


class DiarizerTimeline:
    """One session of a DiarizerTimelines, with the reference's surface (DiarizerTimeline.swift:627-1355)."""

    def __init__(self, timelines: DiarizerTimelines, session: int):
        self.timelines, self.session = timelines, session
        self.config = timelines.config
        self.speakers: dict[int, DiarizerSpeaker] = {}

    def _segments(self, recs, finalized):
        fd = self.config.frame_duration_seconds
        return [DiarizerSegment(int(r["speaker"]), int(r["start_frame"]), int(r["end_frame"]), finalized, fd,
                                float(r["activity"])) for r in recs]

    def _apply(self, fin_recs, ten_recs) -> DiarizerTimelineUpdate:
        for sp in self.speakers.values():
            sp.tentative_segments.clear()
        fin, ten = self._segments(fin_recs, True), self._segments(ten_recs, False)
        if self.config.store_segments:
            # commitSegment (:1315-1324): per speaker in emission order; the lists' speaker-major order keeps it
            for s in fin + ten:
                self.speakers.setdefault(s.speaker_index, DiarizerSpeaker(s.speaker_index)).append(s)
        return DiarizerTimelineUpdate(fin, ten)

    def add_chunk(self, finalized, tentative=()) -> DiarizerTimelineUpdate:
        """addChunk / addPredictions (:801-872): finalized and tentative rows [rows x numSpeakers]"""
        return self.timelines.add_chunks([self], [finalized], [tentative])[0]

    add_predictions = add_chunk

    def finalize(self):
        """finalize (:877-891)"""
        self.timelines.finalize([self.session])
        for sp in self.speakers.values():
            sp.finalize()

    def reset(self, keeping_speakers: bool = False):
        """reset(keepingSpeakers:) (:915-934)"""
        self.timelines.reset([self.session])
        if keeping_speakers:
            for sp in self.speakers.values():
                sp.reset()
        else:
            self.speakers.clear()

    def rebuild(self, finalized, tentative=(), keeping_speakers: bool = False, is_complete: bool = True):
        """rebuild (:945-1003): reset, one push from frame 0 and, when complete, finalize"""
        self.reset(keeping_speakers)
        update = self.add_chunk(finalized, tentative)
        if is_complete:
            self.finalize()
        return update

    def remove_speaker(self, index: int, clear_current_segment: bool = False):
        """removeSpeaker(atIndex:clearCurrentSegment:) (:1125-1139)"""
        if not 0 <= index < self.config.num_speakers:
            return None
        if clear_current_segment:
            self.timelines.clear_speaker(self.session, index)
        return self.speakers.pop(index, None)

    # ---- queries
    def state(self):
        return self.timelines.state(self.session)

    @property
    def num_finalized_frames(self) -> int:
        return self.state().finalized_frames

    @property
    def num_tentative_frames(self) -> int:
        return self.state().tentative.shape[0]

    @property
    def finalized_predictions(self) -> np.ndarray:
        return self.state().stored.reshape(-1)

    @property
    def tentative_predictions(self) -> np.ndarray:
        return self.state().tentative.reshape(-1)

    @property
    def finalized_duration(self) -> float:
        return float(np.float32(self.num_finalized_frames) * np.float32(self.config.frame_duration_seconds))

    def probability(self, speaker: int, frame: int) -> float:
        """probability(speaker:frame:) (:1144-1153): NaN outside the stored frames"""
        st = self.state()
        row = frame - st.finalized_frames + st.stored.shape[0]
        if not (0 <= row < st.stored.shape[0] and speaker < self.config.num_speakers):
            return float("nan")
        return float(st.stored[row, speaker])

    def tentative_probability(self, speaker: int, frame: int) -> float:
        """tentativeProbability(speaker:frame:) (:1156-1165)"""
        st = self.state()
        row = frame - st.finalized_frames
        if not (0 <= row < st.tentative.shape[0] and speaker < self.config.num_speakers):
            return float("nan")
        return float(st.tentative[row, speaker])
