"""Voice activity detection on the GPU (``include/fluidaudio_b200_vad.h``): everything the reference does around the
Silero and FSMN-VAD models (Sources/FluidAudio/VAD/), for many live sessions or clips per call.  The models stay with
the caller.

* ``SileroVadStreams``: live sessions in HBM.  A step is ``model_inputs`` (the 4160-sample model input and the LSTM
  state of every session), the caller's model, then ``advance`` (the new state and streamingStateMachine's events).
* ``segment_speech`` / ``segment_sample_ranges``: segmentSpeech(from:totalSamples:config:) for many clips per call.
* ``fsmn_vad_decide``: FsmnVadManager.decide(silence:) for many clips per call.
* ``VadManager(model=callable)`` mirrors the Swift actor over a batched model callable
  ``model(audio_input [B x 4160], hidden [B x 128], cell [B x 128]) -> (probability [B], new_hidden, new_cell)``.
* ``FsmnVadManager(scorer=callable)`` keeps the reference's chunk schedule on the host around a caller's scorer.

Every config is checked and resolved by ``fa_vad_resolve``; seconds are ``sample / 16000`` and event times round
with Swift's ``.rounded()`` (ties away from zero).
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Callable, List, Optional, Sequence

import numpy as np

from . import _lib

SAMPLE_RATE = 16000
CHUNK_SIZE = 4096          # FA_VAD_CHUNK
CONTEXT_SIZE = 64          # FA_VAD_CONTEXT
STATE_SIZE = 128           # FA_VAD_STATE
MODEL_INPUT_SIZE = 4160    # FA_VAD_MODEL_INPUT
STATUS_OUTPUT_TOO_SMALL = 3
EVENT_NONE, EVENT_START, EVENT_END = 0, 1, 2


@dataclass
class VadConfig:
    default_threshold: float = 0.85


@dataclass
class VadSegmentationConfig:
    min_speech_duration: float = 0.15
    min_silence_duration: float = 0.75
    max_speech_duration: float = 14.0
    speech_padding: float = 0.1
    silence_threshold_for_split: float = 0.3
    negative_threshold: Optional[float] = None
    negative_threshold_offset: float = 0.15
    min_silence_at_max_speech: float = 0.098
    use_max_possible_silence_at_max_speech: bool = True

    def __post_init__(self):
        resolve(VadConfig(), self)   # VadSegmentationConfig.init's preconditions: ValueError here


def _c_config(config: Optional[VadConfig], seg: Optional[VadSegmentationConfig]) -> _lib.VadConfig:
    v = config or VadConfig()
    if seg is None:
        seg = VadSegmentationConfig()
    neg = seg.negative_threshold
    return _lib.VadConfig(v.default_threshold, seg.min_speech_duration, seg.min_silence_duration,
                          seg.max_speech_duration, seg.speech_padding, seg.silence_threshold_for_split,
                          int(neg is not None), 0.0 if neg is None else neg, seg.negative_threshold_offset,
                          seg.min_silence_at_max_speech, int(bool(seg.use_max_possible_silence_at_max_speech)))


def resolve(config: Optional[VadConfig] = None, seg: Optional[VadSegmentationConfig] = None) -> SimpleNamespace:
    """fa_vad_resolve: the working thresholds and sample counts; ValueError for a config the reference traps on"""
    out = _lib.VadResolved()
    st = _lib.load().fa_vad_resolve(C.byref(_c_config(config, seg)), C.byref(out))
    if st != 0:
        raise ValueError(_lib.load().fa_last_error().decode("utf-8", "replace"))
    return SimpleNamespace(**{name: getattr(out, name) for name, _ in out._fields_})


def swift_rounded(x: float) -> float:
    """Double.rounded(): to nearest, ties away from zero"""
    a = abs(x)
    f = math.floor(a)
    return math.copysign(f + 1.0 if a - f >= 0.5 else f, x)


@dataclass
class VadSegment:
    start_time: float
    end_time: float

    @property
    def duration(self) -> float:
        return self.end_time - self.start_time

    def start_sample(self, sample_rate: int = SAMPLE_RATE) -> int:
        return int(self.start_time * float(sample_rate))

    def end_sample(self, sample_rate: int = SAMPLE_RATE) -> int:
        return int(self.end_time * float(sample_rate))

    def sample_count(self, sample_rate: int = SAMPLE_RATE) -> int:
        return self.end_sample(sample_rate) - self.start_sample(sample_rate)


@dataclass
class VadStreamEvent:
    kind: str                     # "speechStart" or "speechEnd"
    sample_index: int
    time: Optional[float] = None

    @property
    def is_start(self) -> bool:
        return self.kind == "speechStart"

    @property
    def is_end(self) -> bool:
        return self.kind == "speechEnd"


def stream_event(kind: int, sample: int, return_seconds: bool = False, time_resolution: int = 1):
    """makeStreamEvent for an advance's (kind, sample); None for no event"""
    if kind == EVENT_NONE:
        return None
    time = None
    if return_seconds:
        factor = math.pow(10.0, float(time_resolution))
        time = swift_rounded(sample / float(SAMPLE_RATE) * factor) / factor
    return VadStreamEvent("speechStart" if kind == EVENT_START else "speechEnd", int(sample), time)


def _offsets(lengths) -> np.ndarray:
    off = np.zeros(len(lengths) + 1, np.int64)
    if len(lengths):
        off[1:] = np.cumsum(lengths)
    return off


class SileroVadStreams:
    """Silero VAD live sessions (fa_vad_stream_*) on the current device"""

    def __init__(self):
        self._L = _lib.load()
        h = C.c_void_p()
        _lib.check(self._L.fa_vad_stream_create(C.byref(h)), "fa_vad_stream_create")
        self._h = h

    def close_handle(self):
        if getattr(self, "_h", None) is not None:
            self._L.fa_vad_stream_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close_handle()
        except Exception:
            pass

    def open(self) -> int:
        sid = C.c_int32()
        _lib.check(self._L.fa_vad_stream_open(self._h, C.byref(sid)), "fa_vad_stream_open")
        return sid.value

    def close(self, session: int):
        _lib.check(self._L.fa_vad_stream_close(self._h, int(session)), "fa_vad_stream_close")

    def model_inputs(self, sessions, chunks):
        """(audio_input [n x 4160], hidden [n x 128], cell [n x 128]) for chunks[i] sent to sessions[i]"""
        ids = np.ascontiguousarray(sessions, np.int32)
        xs = [np.ascontiguousarray(c, np.float32).reshape(-1) for c in chunks]
        audio = np.concatenate(xs) if xs else np.zeros(0, np.float32)
        off = _offsets([x.size for x in xs])
        n = ids.size
        inp = np.empty((n, MODEL_INPUT_SIZE), np.float32)
        hid, cel = np.empty((n, STATE_SIZE), np.float32), np.empty((n, STATE_SIZE), np.float32)
        _lib.check(self._L.fa_vad_stream_model_inputs(self._h, n, _lib.ptr(ids), _lib.ptr(audio), _lib.ptr(off),
                                                      _lib.ptr(inp), _lib.ptr(hid), _lib.ptr(cel)),
                   "fa_vad_stream_model_inputs")
        return inp, hid, cel

    def model_inputs_device(self, sessions, d_audio: "_lib.DeviceBuffer", offsets, d_audio_input: "_lib.DeviceBuffer",
                            d_hidden: "_lib.DeviceBuffer", d_cell: "_lib.DeviceBuffer"):
        ids = np.ascontiguousarray(sessions, np.int32)
        off = np.ascontiguousarray(offsets, np.int64)
        _lib.check(self._L.fa_vad_stream_model_inputs_device(self._h, ids.size, _lib.ptr(ids), d_audio.ptr,
                                                             _lib.ptr(off), d_audio_input.ptr, d_hidden.ptr,
                                                             d_cell.ptr), "fa_vad_stream_model_inputs_device")

    def advance(self, sessions, probability, new_hidden, new_cell, config: Optional[VadConfig] = None,
                seg: Optional[VadSegmentationConfig] = None) -> np.ndarray:
        """commits the staged chunks; events [n x 2] as (kind, sample): kind 0 none, 1 start, 2 end"""
        ids = np.ascontiguousarray(sessions, np.int32)
        p = np.ascontiguousarray(probability, np.float32).reshape(-1)
        h = np.ascontiguousarray(new_hidden, np.float32)
        c = np.ascontiguousarray(new_cell, np.float32)
        ev = np.empty((ids.size, 2), np.int64)
        cfg = _c_config(config, seg)
        _lib.check(self._L.fa_vad_stream_advance(self._h, ids.size, _lib.ptr(ids), _lib.ptr(p), _lib.ptr(h),
                                                 _lib.ptr(c), C.byref(cfg), _lib.ptr(ev)), "fa_vad_stream_advance")
        return ev

    def advance_device(self, sessions, d_probability, d_new_hidden, d_new_cell, d_events,
                       config: Optional[VadConfig] = None, seg: Optional[VadSegmentationConfig] = None):
        ids = np.ascontiguousarray(sessions, np.int32)
        cfg = _c_config(config, seg)
        _lib.check(self._L.fa_vad_stream_advance_device(self._h, ids.size, _lib.ptr(ids), d_probability.ptr,
                                                        d_new_hidden.ptr, d_new_cell.ptr, C.byref(cfg), d_events.ptr),
                   "fa_vad_stream_advance_device")

    def state(self, session: int) -> SimpleNamespace:
        """VadStreamState of the session: context, hidden, cell, triggered, temp_end_sample (None: nil),
        processed_samples, and whether a staged chunk waits for its advance"""
        info = _lib.VadSessionInfo()
        ctx, hid = np.empty(CONTEXT_SIZE, np.float32), np.empty(STATE_SIZE, np.float32)
        cel = np.empty(STATE_SIZE, np.float32)
        _lib.check(self._L.fa_vad_stream_session_state(self._h, int(session), C.byref(info), _lib.ptr(ctx),
                                                       _lib.ptr(hid), _lib.ptr(cel)), "fa_vad_stream_session_state")
        return SimpleNamespace(context=ctx, hidden=hid, cell=cel, triggered=bool(info.triggered),
                               temp_end_sample=None if info.temp_end_sample < 0 else int(info.temp_end_sample),
                               processed_samples=int(info.processed_samples), has_pending=bool(info.has_pending))


def _clip_call(name, inputs, extra, capacity=None):
    xs = [np.ascontiguousarray(x, np.float32).reshape(-1) for x in inputs]
    data = np.concatenate(xs) if xs else np.zeros(0, np.float32)
    off = _offsets([x.size for x in xs])
    counts = np.zeros(len(xs), np.int64)
    total = C.c_int64()
    L = _lib.load()
    cap = sum(x.size for x in xs) if capacity is None else int(capacity)
    seg = np.zeros((max(cap, 1), 2), np.int64)
    st = getattr(L, name)(_lib.ptr(data), _lib.ptr(off), len(xs), *extra(len(xs)), _lib.ptr(counts), _lib.ptr(seg),
                          cap, C.byref(total))
    _lib.check(st, name)
    out, at = [], 0
    for n in counts:
        out.append(seg[at:at + n].copy())
        at += n
    return out


def segment_sample_ranges(probabilities: Sequence, total_samples: Sequence[int], config: Optional[VadConfig] = None,
                          seg: Optional[VadSegmentationConfig] = None) -> List[np.ndarray]:
    """Per clip, its speech sample ranges [n x 2] (start, end) from its per-chunk probabilities"""
    ts = np.ascontiguousarray(total_samples, np.int64).reshape(-1)
    if ts.size != len(probabilities):
        raise ValueError(f"{ts.size} total_samples for {len(probabilities)} clips")
    cfg = _c_config(config, seg)
    return _clip_call("fa_vad_segment", probabilities, lambda n: (_lib.ptr(ts), C.byref(cfg)))


def segment_speech(probabilities: Sequence, total_samples: Sequence[int], config: Optional[VadConfig] = None,
                   seg: Optional[VadSegmentationConfig] = None) -> List[List[VadSegment]]:
    """segmentSpeech(from:totalSamples:config:) for many clips: per clip, its VadSegments in seconds"""
    return [[VadSegment(int(a) / float(SAMPLE_RATE), int(b) / float(SAMPLE_RATE)) for a, b in r]
            for r in segment_sample_ranges(probabilities, total_samples, config, seg)]


@dataclass
class FsmnVadSegment:
    start_ms: int
    end_ms: int


def fsmn_vad_decide(silences: Sequence) -> List[List[FsmnVadSegment]]:
    """FsmnVadManager.decide(silence:) for many clips of per-frame silence probabilities"""
    return [[FsmnVadSegment(int(a), int(b)) for a, b in r]
            for r in _clip_call("fa_fsmn_vad_decide", silences, lambda n: (), None)]


@dataclass
class VadStreamResult:
    session: int
    event: Optional[VadStreamEvent]
    probability: float


class VadManager:
    """VadManager over a batched model callable (see the module docstring); its sessions live in one
    SileroVadStreams"""

    sample_rate = SAMPLE_RATE
    chunk_size = CHUNK_SIZE

    def __init__(self, model: Callable, config: Optional[VadConfig] = None):
        self.model = model
        self.config = config or VadConfig()
        self.streams = SileroVadStreams()

    def _step(self, sessions, chunks):
        inp, hid, cel = self.streams.model_inputs(sessions, chunks)
        p, h, c = self.model(inp, hid, cel)
        return np.asarray(p, np.float32).reshape(-1), np.asarray(h, np.float32), np.asarray(c, np.float32)

    def process(self, clips) -> List[np.ndarray]:
        """processAudioSamples for many clips at once: per clip, the probability of each 4096-sample chunk"""
        xs = [np.asarray(c, np.float32).reshape(-1) for c in clips]
        ids = [self.streams.open() for _ in xs]
        try:
            out = [np.zeros((x.size + CHUNK_SIZE - 1) // CHUNK_SIZE, np.float32) for x in xs]
            k = 0
            while True:
                live = [i for i, x in enumerate(xs) if x.size > k * CHUNK_SIZE]
                if not live:
                    break
                sess = [ids[i] for i in live]
                p, h, c = self._step(sess, [xs[i][k * CHUNK_SIZE:(k + 1) * CHUNK_SIZE] for i in live])
                self.streams.advance(sess, p, h, c, self.config)
                for j, i in enumerate(live):
                    out[i][k] = p[j]
                k += 1
            return out
        finally:
            for s in ids:
                self.streams.close(s)

    def make_stream_state(self) -> int:
        """a fresh session (VadStreamState.initial()); close it with close_stream_state"""
        return self.streams.open()

    def close_stream_state(self, session: int):
        self.streams.close(session)

    def process_streaming_chunk(self, chunk, session: int, config: Optional[VadSegmentationConfig] = None,
                                return_seconds: bool = False, time_resolution: int = 1) -> VadStreamResult:
        """processStreamingChunk on one session (its state stays in HBM; see SileroVadStreams.state)"""
        p, h, c = self._step([session], [chunk])
        ev = self.streams.advance([session], p, h, c, self.config, config)
        return VadStreamResult(session, stream_event(int(ev[0, 0]), int(ev[0, 1]), return_seconds, time_resolution),
                               float(p[0]))

    def segment_speech_from(self, probabilities, total_samples: int,
                            config: Optional[VadSegmentationConfig] = None) -> List[VadSegment]:
        """segmentSpeech(from:totalSamples:config:) over one clip's chunk probabilities"""
        return segment_speech([probabilities], [total_samples], self.config, config)[0]

    def segment_speech(self, samples, config: Optional[VadSegmentationConfig] = None) -> List[VadSegment]:
        x = np.asarray(samples, np.float32).reshape(-1)
        return self.segment_speech_from(self.process([x])[0], x.size, config)

    def segment_speech_audio(self, samples, config: Optional[VadSegmentationConfig] = None) -> List[np.ndarray]:
        """each segment's samples, sliced at Int(startTime * 16000) as the reference slices"""
        x = np.asarray(samples, np.float32).reshape(-1)
        out = []
        for s in self.segment_speech(x, config):
            a = max(0, min(s.start_sample(), x.size))
            b = max(a, min(s.end_sample(), x.size))
            out.append(x[a:b].copy())
        return out


class FsmnVadManager:
    """FsmnVadManager's host side: the chunk schedule (concatenateChunks, lfrFrameCount) around a caller's scorer
    ``scorer(samples) -> silence probabilities`` (the x32768 scaling, preprocessor and FSMN model), and the decision
    on the GPU"""

    BUCKETS = (512, 1024, 2048, 3072)
    HOP_SAMPLES = 160
    FBANK_WINDOW_SAMPLES = 400
    LFR_PAD_FRAMES = 2
    LFR_WIDTH = 5
    WINDOW_FRAMES = 20

    def __init__(self, scorer: Callable):
        self.scorer = scorer

    @staticmethod
    def concatenate_chunks(sample_count: int, score: Callable) -> np.ndarray:
        """concatenateChunks (FsmnVadManager.swift:91-109): score(start, end) for each chunk, frames on the 10 ms grid"""
        chunk = (FsmnVadManager.BUCKETS[-1] - FsmnVadManager.WINDOW_FRAMES) * FsmnVadManager.HOP_SAMPLES
        parts, kept, start = [], 0, 0
        while start < sample_count:
            end = min(start + chunk, sample_count)
            sil = np.asarray(score(start, end), np.float32).reshape(-1)
            keep = 0 if start == 0 else FsmnVadManager.LFR_PAD_FRAMES
            if sil.size <= keep:
                break
            parts.append(sil[keep:])
            kept += sil.size - keep
            if end == sample_count:
                break
            start = (kept - FsmnVadManager.LFR_PAD_FRAMES) * FsmnVadManager.HOP_SAMPLES
        return np.concatenate(parts) if parts else np.zeros(0, np.float32)

    @staticmethod
    def lfr_frame_count(samples: int) -> int:
        """lfrFrameCount (:113-117)"""
        if samples < FsmnVadManager.FBANK_WINDOW_SAMPLES:
            return 0
        fbank = (samples - FsmnVadManager.FBANK_WINDOW_SAMPLES) // FsmnVadManager.HOP_SAMPLES + 1
        return max(0, fbank + FsmnVadManager.LFR_PAD_FRAMES - FsmnVadManager.LFR_WIDTH + 1)

    def silence_probabilities(self, audio) -> np.ndarray:
        x = np.asarray(audio, np.float32).reshape(-1)
        return self.concatenate_chunks(x.size, lambda a, b: self.scorer(x[a:b]))

    def detect(self, audio) -> List[FsmnVadSegment]:
        return fsmn_vad_decide([self.silence_probabilities(audio)])[0]

    def detect_many(self, clips) -> List[List[FsmnVadSegment]]:
        """detect for many clips, their decisions in one call"""
        return fsmn_vad_decide([self.silence_probabilities(c) for c in clips])
