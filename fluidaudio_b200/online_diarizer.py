"""Streaming speaker tracking for many live sessions: DiarizerManager's chunk logic and SpeakerManager's speaker
database (include/fluidaudio_b200_online_diar.h).  The segmentation and embedding models stay with the caller.

A chunk of every session is three calls around the two models:

    seg, wave = chunk_inputs(chunks, config)                 # the models' waveforms
    masks, need = dbs.embedding_inputs(sessions, logits)     # after the segmentation model
    assigned, segments = dbs.advance(sessions, embeddings, offsets)   # after the embedding model

Speaker ids are strings.  A canonical decimal id (what ``str(int(s)) == s`` holds for, and what every speaker the
tracker creates has) travels as (0, value); any other string travels as (1, key) with a key this module assigns.
"""
from __future__ import annotations

import ctypes as C
import re
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib

DIM, FIFO, CLASSES, LOCAL, MODEL_SAMPLES = 256, 50, 7, 3, 160000
MODES = {"reset": 0, "merge": 1, "overwrite": 2, "skip": 3}
_INT = re.compile(r"[+-]?[0-9]+\Z")


@dataclass
class DiarizerConfig:
    """DiarizerConfig with the reference defaults"""
    clustering_threshold: float = 0.7
    min_speech_duration: float = 1.0
    min_embedding_update_duration: float = 2.0
    min_silence_gap: float = 0.5
    num_clusters: int = -1
    min_active_frames_count: float = 10.0
    chunk_duration: float = 10.0
    chunk_overlap: float = 0.0

    def c(self) -> _lib.OnlineDiarConfig:
        return _lib.OnlineDiarConfig(self.clustering_threshold, self.min_speech_duration,
                                     self.min_embedding_update_duration, self.min_silence_gap, self.num_clusters,
                                     self.min_active_frames_count, self.chunk_duration, self.chunk_overlap)


def resolve(config: Optional[DiarizerConfig] = None) -> _lib.OnlineDiarResolved:
    out = _lib.OnlineDiarResolved()
    _lib.check(_lib.load().fa_od_resolve(C.byref((config or DiarizerConfig()).c()), C.byref(out)), "fa_od_resolve")
    return out


def swift_int(s: str) -> Optional[int]:
    """Int(s) in Swift: an optional sign and ASCII digits, inside Int64"""
    if not _INT.match(s):
        return None
    v = int(s)
    return v if -(1 << 63) <= v < (1 << 63) else None


def _offsets(clips: Sequence[np.ndarray]):
    lens = [len(c) for c in clips]
    off = np.zeros(len(clips) + 1, np.int64)
    off[1:] = np.cumsum(lens)
    audio = np.concatenate([np.asarray(c, np.float32) for c in clips]) if sum(lens) else np.zeros(0, np.float32)
    return np.ascontiguousarray(audio), off


def chunk_inputs(chunks: Sequence[np.ndarray], config: Optional[DiarizerConfig] = None):
    """(segmentation inputs, embedding waveforms), each [len(chunks) x 160000]"""
    audio, off = _offsets(chunks)
    n = len(chunks)
    seg, wave = np.empty((n, MODEL_SAMPLES), np.float32), np.empty((n, MODEL_SAMPLES), np.float32)
    _lib.check(_lib.load().fa_od_chunk_inputs(_lib.ptr(audio) if audio.size else None, off.ctypes.data, n,
                                              resolve(config).chunk_size, seg.ctypes.data, wave.ctypes.data),
               "fa_od_chunk_inputs")
    return seg, wave


def enrollment_inputs(clips: Sequence[np.ndarray], frames: int = 589):
    """extractSpeakerEmbedding(from:)'s (waveforms [n x 160000], masks [n x frames])"""
    audio, off = _offsets(clips)
    n = len(clips)
    wave, mask = np.empty((n, MODEL_SAMPLES), np.float32), np.empty((n, frames), np.float32)
    _lib.check(_lib.load().fa_od_enrollment_inputs(_lib.ptr(audio) if audio.size else None, off.ctypes.data, n,
                                                   frames, wave.ctypes.data, mask.ctypes.data),
               "fa_od_enrollment_inputs")
    return wave, mask


@dataclass
class Speaker:
    """A known speaker as SpeakerManager takes it: Speaker.init normalises current_embedding, RawEmbedding.init each
    raw row"""
    id: str
    current_embedding: np.ndarray
    duration: float = 0.0
    update_count: int = 1
    raw_embeddings: Optional[np.ndarray] = None
    is_permanent: bool = False


@dataclass
class SpeakerState:
    """One speaker as a session's database holds it"""
    id: str
    current_embedding: np.ndarray
    duration: float
    update_count: int
    raw_embeddings: np.ndarray
    is_permanent: bool


@dataclass
class TimedSpeakerSegment:
    speaker_id: str
    start_time_seconds: float
    end_time_seconds: float
    quality_score: float


class SpeakerDatabases:
    """Live sessions, each one SpeakerManager with DiarizerManager's chunk state, in HBM"""

    def __init__(self, frames: int = 589, config: Optional[DiarizerConfig] = None):
        self.frames = int(frames)
        self.config = config or DiarizerConfig()
        self._L = _lib.load()
        h = C.c_void_p()
        _lib.check(self._L.fa_od_create(self.frames, C.byref(h)), "fa_od_create")
        self._h = h
        self._names: Dict[str, int] = {}
        self._by_key: Dict[int, str] = {}

    def close_handle(self) -> None:
        if self._h is not None:
            self._L.fa_od_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close_handle()
        except Exception:
            pass

    # ---- identities
    def identity(self, sid: str) -> Tuple[int, int]:
        v = swift_int(sid)
        if v is not None and str(v) == sid:
            return 0, v
        if sid not in self._names:
            self._names[sid] = len(self._names)
            self._by_key[self._names[sid]] = sid
        return 1, self._names[sid]

    def name(self, named: int, key: int) -> str:
        return "" if named < 0 else str(int(key)) if named == 0 else self._by_key[int(key)]

    # ---- sessions
    def open(self) -> int:
        s = C.c_int32()
        _lib.check(self._L.fa_od_open(self._h, C.byref(s)), "fa_od_open")
        return s.value

    def close(self, session: int) -> None:
        _lib.check(self._L.fa_od_close(self._h, session), "fa_od_close")

    def embedding_inputs(self, sessions: Sequence[int], logits: np.ndarray):
        """logits [n x F x 7] -> (masks [n x 3 x F], need [n x 3])"""
        s = np.ascontiguousarray(sessions, np.int32)
        lg = np.ascontiguousarray(logits, np.float32).reshape(len(s), self.frames, CLASSES)
        masks, need = np.empty((len(s), LOCAL, self.frames), np.float32), np.empty((len(s), LOCAL), np.int32)
        _lib.check(self._L.fa_od_embedding_inputs(self._h, len(s), s.ctypes.data, lg.ctypes.data,
                                                  C.byref(self.config.c()), masks.ctypes.data, need.ctypes.data),
                   "fa_od_embedding_inputs")
        return masks, need

    def advance_raw(self, sessions: Sequence[int], embeddings: np.ndarray, offsets: Sequence[float]):
        """(assigned [n x 3 x 2], counts [n], ids [n x bound x 2], values [n x bound x 3]) as the C ABI writes them"""
        s = np.ascontiguousarray(sessions, np.int32)
        n, bound = len(s), 3 * ((self.frames + 1) // 2)
        e = np.ascontiguousarray(embeddings, np.float32).reshape(n, LOCAL, DIM)
        off = np.ascontiguousarray(offsets, np.float64)
        assigned = np.empty((n, LOCAL, 2), np.int64)
        counts = np.empty(n, np.int32)
        ids, vals = np.empty((n, bound, 2), np.int64), np.empty((n, bound, 3), np.float32)
        _lib.check(self._L.fa_od_advance(self._h, n, s.ctypes.data, e.ctypes.data, off.ctypes.data,
                                         C.byref(self.config.c()), assigned.ctypes.data, counts.ctypes.data,
                                         ids.ctypes.data, vals.ctypes.data), "fa_od_advance")
        return assigned, counts, ids, vals

    def advance(self, sessions: Sequence[int], embeddings: np.ndarray, offsets: Sequence[float]):
        """(speaker ids [n][3] ("" for none), segments [n][...])"""
        assigned, counts, ids, vals = self.advance_raw(sessions, embeddings, offsets)
        names = [[self.name(*a) for a in row] for row in assigned]
        segs = [[TimedSpeakerSegment(self.name(*ids[b, k]), float(vals[b, k, 0]), float(vals[b, k, 1]),
                                     float(vals[b, k, 2])) for k in range(counts[b])] for b in range(len(counts))]
        return names, segs

    # ---- the database
    def read_raw(self, session: int):
        c, nx = C.c_int64(), C.c_int64()
        _lib.check(self._L.fa_od_speaker_count(self._h, session, C.byref(c), C.byref(nx)), "fa_od_speaker_count")
        sp = np.zeros(c.value, _lib.ONLINE_DIAR_SPEAKER)
        cur, raws = np.zeros((c.value, DIM), np.float32), np.zeros((c.value, FIFO, DIM), np.float32)
        _lib.check(self._L.fa_od_read(self._h, session, sp.ctypes.data, cur.ctypes.data, raws.ctypes.data),
                   "fa_od_read")
        return sp, cur, raws, nx.value

    def speakers(self, session: int) -> List[SpeakerState]:
        sp, cur, raws, _ = self.read_raw(session)
        return [SpeakerState(self.name(int(s["named"]), int(s["key"])), cur[i], float(s["duration"]),
                             int(s["update_count"]), raws[i, :s["raw_count"]], bool(s["permanent"]))
                for i, s in enumerate(sp)]

    def initialize_known_speakers(self, session: int, speakers: Sequence[Speaker], mode: str = "skip",
                                  preserve_if_permanent: bool = True) -> None:
        sp = np.zeros(len(speakers), _lib.ONLINE_DIAR_SPEAKER)
        rows = []
        for i, k in enumerate(speakers):
            named, key = self.identity(k.id)
            v = swift_int(k.id)
            raws = np.zeros((0, DIM), np.float32) if k.raw_embeddings is None else np.asarray(k.raw_embeddings, np.float32)
            sp[i] = (key, v or 0, k.update_count, k.duration, named, v is not None, k.is_permanent, len(raws))
            rows.append(raws.reshape(-1, DIM))
        cur = np.ascontiguousarray(np.array([k.current_embedding for k in speakers], np.float32).reshape(-1, DIM))
        raw = np.ascontiguousarray(np.concatenate(rows) if rows else np.zeros((0, DIM), np.float32))
        _lib.check(self._L.fa_od_initialize(self._h, session, len(sp), sp.ctypes.data, cur.ctypes.data,
                                            raw.ctypes.data if raw.size else None, MODES[mode],
                                            int(preserve_if_permanent)), "fa_od_initialize")

    def remove_speaker(self, session: int, sid: str, keep_if_permanent: bool = True) -> bool:
        out = C.c_int32()
        _lib.check(self._L.fa_od_remove(self._h, session, *self.identity(sid), int(keep_if_permanent),
                                        C.byref(out)), "fa_od_remove")
        return bool(out.value)

    def merge_speaker(self, session: int, source: str, destination: str, stop_if_permanent: bool = True) -> bool:
        out = C.c_int32()
        _lib.check(self._L.fa_od_merge(self._h, session, *self.identity(source), *self.identity(destination),
                                       int(stop_if_permanent), C.byref(out)), "fa_od_merge")
        return bool(out.value)

    def set_permanent(self, session: int, sid: str, permanent: bool = True) -> bool:
        out = C.c_int32()
        _lib.check(self._L.fa_od_set_permanent(self._h, session, *self.identity(sid), int(permanent),
                                               C.byref(out)), "fa_od_set_permanent")
        return bool(out.value)

    def reset(self, session: int, keep_if_permanent: bool = False) -> None:
        _lib.check(self._L.fa_od_reset(self._h, session, int(keep_if_permanent)), "fa_od_reset")

    def distances(self, session: int, embeddings: np.ndarray) -> np.ndarray:
        e = np.ascontiguousarray(embeddings, np.float32).reshape(-1, DIM)
        c, nx = C.c_int64(), C.c_int64()
        _lib.check(self._L.fa_od_speaker_count(self._h, session, C.byref(c), C.byref(nx)), "fa_od_speaker_count")
        out = np.zeros((len(e), c.value), np.float32)
        _lib.check(self._L.fa_od_query(self._h, session, len(e), e.ctypes.data, out.ctypes.data), "fa_od_query")
        return out

    def find_speaker(self, session: int, embeddings: np.ndarray, threshold: Optional[float] = None):
        """findSpeaker for each embedding: (id or None, distance or inf); ties go to the earlier speaker"""
        thr = np.float32(resolve(self.config).speaker_threshold if threshold is None else threshold)
        ids = [s.id for s in self.speakers(session)]
        out = []
        for row in self.distances(session, embeddings):
            best, at = np.float32(np.inf), -1
            for i, d in enumerate(row):
                if d < best:
                    best, at = d, i
            out.append((ids[at], float(best)) if at >= 0 and best <= thr else (None, float("inf")))
        return out

    def find_matching_speakers(self, session: int, embedding: np.ndarray, threshold: Optional[float] = None):
        """findMatchingSpeakers: every speaker within the threshold (<=), by distance, ties in database order"""
        thr = np.float32(resolve(self.config).speaker_threshold if threshold is None else threshold)
        ids = [s.id for s in self.speakers(session)]
        row = self.distances(session, embedding)[0]
        hits = [(ids[i], float(d)) for i, d in enumerate(row) if d <= thr]
        return sorted(hits, key=lambda t: t[1])

    def upsert_speaker(self, session: int, speaker: Speaker) -> None:
        """upsertSpeaker: an existing id takes the fields as given, a new one is Speaker.init of them"""
        named, key = self.identity(speaker.id)
        v = swift_int(speaker.id)
        raws = np.zeros((0, DIM), np.float32) if speaker.raw_embeddings is None else \
            np.ascontiguousarray(np.asarray(speaker.raw_embeddings, np.float32).reshape(-1, DIM))
        sp = np.zeros(1, _lib.ONLINE_DIAR_SPEAKER)
        sp[0] = (key, v or 0, speaker.update_count, speaker.duration, named, v is not None, speaker.is_permanent,
                 len(raws))
        cur = np.ascontiguousarray(speaker.current_embedding, np.float32)
        _lib.check(self._L.fa_od_upsert(self._h, session, sp.ctypes.data, cur.ctypes.data,
                                        raws.ctypes.data if raws.size else None), "fa_od_upsert")

    def find_mergeable_pairs(self, session: int, threshold: Optional[float] = None,
                             exclude_if_both_permanent: bool = True) -> List[Tuple[str, str]]:
        """findMergeablePairs over the database in insertion order: (speaker to merge, destination)"""
        thr = np.float32(resolve(self.config).speaker_threshold if threshold is None else threshold)
        sp = self.speakers(session)
        if not sp:
            return []
        dist = self.distances(session, np.stack([s.current_embedding for s in sp]))
        pairs = []
        for i in range(len(sp)):
            for j in range(i + 1, len(sp)):
                if exclude_if_both_permanent and sp[i].is_permanent and sp[j].is_permanent:
                    continue
                if not dist[i, j] < thr:
                    continue
                pairs.append((sp[j].id, sp[i].id) if not sp[j].is_permanent else (sp[i].id, sp[j].id))
        return pairs


class SpeakerManager:
    """SpeakerManager's public interface over one session of a SpeakerDatabases"""

    def __init__(self, config: Optional[DiarizerConfig] = None, frames: int = 589,
                 databases: Optional[SpeakerDatabases] = None):
        self.dbs = databases or SpeakerDatabases(frames, config)
        self.session = self.dbs.open()

    def initialize_known_speakers(self, speakers, mode="skip", preserve_if_permanent=True):
        self.dbs.initialize_known_speakers(self.session, speakers, mode, preserve_if_permanent)

    def upsert_speaker(self, speaker: Speaker):
        self.dbs.upsert_speaker(self.session, speaker)

    def remove_speaker(self, sid: str, keep_if_permanent: bool = True) -> bool:
        return self.dbs.remove_speaker(self.session, sid, keep_if_permanent)

    def merge_speaker(self, source: str, destination: str, stop_if_permanent: bool = True) -> bool:
        return self.dbs.merge_speaker(self.session, source, destination, stop_if_permanent)

    def make_speaker_permanent(self, sid: str) -> bool:
        return self.dbs.set_permanent(self.session, sid, True)

    def revoke_permanence(self, sid: str) -> bool:
        return self.dbs.set_permanent(self.session, sid, False)

    def reset(self, keep_if_permanent: bool = False):
        self.dbs.reset(self.session, keep_if_permanent)

    def find_speaker(self, embedding, threshold=None):
        return self.dbs.find_speaker(self.session, embedding, threshold)[0]

    def find_matching_speakers(self, embedding, threshold=None):
        return self.dbs.find_matching_speakers(self.session, embedding, threshold)

    def find_mergeable_pairs(self, threshold=None, exclude_if_both_permanent=True):
        return self.dbs.find_mergeable_pairs(self.session, threshold, exclude_if_both_permanent)

    def get_all_speakers(self) -> Dict[str, SpeakerState]:
        return {s.id: s for s in self.dbs.speakers(self.session)}

    @property
    def speaker_count(self) -> int:
        return len(self.dbs.speakers(self.session))


class DiarizerManager:
    """DiarizerManager with the two models as callables:
    segmentation_model(waveforms [n x 160000]) -> logits [n x F x 7];
    embedding_model(waveforms [n x 160000], masks [n x F]) -> embeddings [n x 256]."""

    def __init__(self, segmentation_model, embedding_model, config: Optional[DiarizerConfig] = None,
                 frames: int = 589):
        self.config = config or DiarizerConfig()
        self.segmentation_model, self.embedding_model = segmentation_model, embedding_model
        self.speaker_manager = SpeakerManager(self.config, frames)
        self.frames = frames

    def extract_speaker_embedding(self, audio: np.ndarray) -> np.ndarray:
        wave, mask = enrollment_inputs([audio], self.frames)
        return np.asarray(self.embedding_model(wave, mask), np.float32)[0]

    def perform_complete_diarization(self, samples: np.ndarray, start_time: float = 0.0,
                                     sample_rate: int = 16000) -> List[TimedSpeakerSegment]:
        r = resolve(self.config)
        dbs, sid = self.speaker_manager.dbs, self.speaker_manager.session
        samples = np.asarray(samples, np.float32)
        out: List[TimedSpeakerSegment] = []
        if r.step_size <= 0:
            return out
        for at in range(0, len(samples), r.step_size):
            seg, wave = chunk_inputs([samples[at:at + r.chunk_size]], self.config)
            logits = np.asarray(self.segmentation_model(seg), np.float32)
            masks, need = dbs.embedding_inputs([sid], logits)
            emb = np.zeros((1, LOCAL, DIM), np.float32)
            for s in range(LOCAL):
                if need[0, s]:
                    emb[0, s] = np.asarray(self.embedding_model(wave, masks[:, s]), np.float32)[0]
            _, segs = dbs.advance([sid], emb, [at / sample_rate + start_time])
            out.extend(segs[0])
        return out
