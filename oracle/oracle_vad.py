"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.

ctypes front-end to ``liboracle_vad.so``, the sequential CPU restatement of voice activity detection around the
Silero and FSMN-VAD models (``oracle_vad.cpp``: the config checks and thresholds, processChunk's staging,
streamingStateMachine, detectSpeechSampleRanges with its whole possibleEnds list, FsmnVadManager.decide), compiled
into its own library with the main oracle's pinned flags (``-O2 -ffp-contract=off`` on baseline x86-64).
Importers allowed: ``tests/``, ``__graft_entry__`` and ``scripts/``.  The product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "oracle_vad.cpp")]
_LIB = os.path.join(_HERE, "liboracle_vad.so")
_FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-Wall", "-Wextra", "-shared"]

CHUNK, CONTEXT, STATE = 4096, 64, 128

_lib = None


class Config(C.Structure):
    """fa_vad_config's layout"""
    _fields_ = [("default_threshold", C.c_float), ("min_speech_duration", C.c_double),
                ("min_silence_duration", C.c_double), ("max_speech_duration", C.c_double),
                ("speech_padding", C.c_double), ("silence_threshold_for_split", C.c_float),
                ("has_negative_threshold", C.c_int32), ("negative_threshold", C.c_float),
                ("negative_threshold_offset", C.c_float), ("min_silence_at_max_speech", C.c_double),
                ("use_max_possible_silence_at_max_speech", C.c_int32)]


class Resolved(C.Structure):
    """fa_vad_resolved's layout"""
    _fields_ = [("threshold", C.c_float), ("negative_threshold", C.c_float),
                ("silence_threshold_for_split", C.c_float), ("use_max_possible_silence_at_max_speech", C.c_int32),
                ("min_speech_samples", C.c_int64), ("min_silence_samples", C.c_int64),
                ("max_speech_samples", C.c_int64), ("speech_pad_samples", C.c_int64),
                ("min_silence_at_max_speech_samples", C.c_int64)]


def config(default_threshold=0.85, min_speech_duration=0.15, min_silence_duration=0.75, max_speech_duration=14.0,
           speech_padding=0.1, silence_threshold_for_split=0.3, negative_threshold=None,
           negative_threshold_offset=0.15, min_silence_at_max_speech=0.098,
           use_max_possible_silence_at_max_speech=True) -> Config:
    """VadConfig.defaultThreshold and VadSegmentationConfig with the reference defaults"""
    return Config(default_threshold, min_speech_duration, min_silence_duration, max_speech_duration, speech_padding,
                  silence_threshold_for_split, int(negative_threshold is not None),
                  0.0 if negative_threshold is None else negative_threshold, negative_threshold_offset,
                  min_silence_at_max_speech, int(bool(use_max_possible_silence_at_max_speech)))


def build(force: bool = False) -> None:
    """Compile liboracle_vad.so when it is missing or older than a source."""
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in _SRCS):
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx, *_FLAGS, "-o", _LIB, *_SRCS])


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        vp, i64, f32 = C.c_void_p, C.c_int64, C.c_float
        L.oracle_vad_resolve.argtypes = [C.POINTER(Config), C.POINTER(Resolved)]
        L.oracle_vad_resolve.restype = C.c_int
        L.oracle_vad_model_input.argtypes = [vp, vp, i64, vp, vp]
        L.oracle_vad_model_input.restype = None
        L.oracle_vad_stream_step.argtypes = [vp, f32, i64, C.POINTER(Resolved), C.POINTER(i64)]
        L.oracle_vad_stream_step.restype = C.c_int
        L.oracle_vad_segment.argtypes = [vp, i64, i64, C.POINTER(Resolved), vp, i64]
        L.oracle_vad_segment.restype = i64
        L.oracle_vad_tick.argtypes = [i64] + [vp] * 9 + [C.POINTER(Resolved)] + [vp] * 4
        L.oracle_vad_tick.restype = None
        L.oracle_vad_segment_batch.argtypes = [vp, vp, i64, vp, C.POINTER(Resolved), vp, vp]
        L.oracle_vad_segment_batch.restype = i64
        L.oracle_fsmn_decide.argtypes = [vp, i64, vp, i64]
        L.oracle_fsmn_decide.restype = i64
        _lib = L
    return _lib


def resolve(cfg: Config):
    """the resolved config, or None when it is refused"""
    r = Resolved()
    return r if lib().oracle_vad_resolve(C.byref(cfg), C.byref(r)) == 0 else None


def _resolved(cfg):
    r = resolve(cfg) if isinstance(cfg, Config) else cfg
    assert r is not None, "the config is refused"
    return r


def model_input(context, chunk):
    """(audio_input [4160], next context [64]) of processChunk"""
    ctx = np.ascontiguousarray(context, np.float32)
    x = np.ascontiguousarray(chunk, np.float32).reshape(-1)
    inp, nxt = np.zeros(CHUNK + CONTEXT, np.float32), np.zeros(CONTEXT, np.float32)
    lib().oracle_vad_model_input(ctx.ctypes.data, x.ctypes.data if x.size else None, x.size, inp.ctypes.data,
                                 nxt.ctypes.data)
    return inp, nxt


class Stream:
    """VadStreamState and streamingStateMachine, with the model's state carried as the reference carries it"""

    def __init__(self):
        self.state = np.array([0, 0, -1], np.int64)   # processedSamples, triggered, tempEndSample (-1 nil)
        self.context = np.zeros(CONTEXT, np.float32)
        self.hidden = np.zeros(STATE, np.float32)
        self.cell = np.zeros(STATE, np.float32)

    def step(self, probability, chunk_count, cfg):
        """(kind, sample) of one committed chunk: kind 0 none (sample -1), 1 start, 2 end"""
        sample = C.c_int64()
        r = _resolved(cfg)
        kind = lib().oracle_vad_stream_step(self.state.ctypes.data, np.float32(probability), int(chunk_count),
                                            C.byref(r), C.byref(sample))
        return int(kind), int(sample.value)

    def chunk(self, chunk, model, cfg):
        """processStreamingChunk with a batched model (see _one): (kind, sample, probability)"""
        inp, nxt = model_input(self.context, chunk)
        p, h, c = _one(model, inp, self.hidden, self.cell)
        self.hidden, self.cell, self.context = h, c, nxt
        return self.step(p, len(chunk), cfg) + (p,)


def _one(model, inp, hidden, cell):
    """a batched model(audio_input [B x 4160], hidden [B x 128], cell [B x 128]) on one row"""
    p, h, c = model(inp[None].copy(), hidden[None].copy(), cell[None].copy())
    return (np.float32(np.asarray(p, np.float32).reshape(-1)[0]), np.asarray(h, np.float32).reshape(-1).copy(),
            np.asarray(c, np.float32).reshape(-1).copy())


def process(audio, model):
    """processAudioSamples with a batched model (see _one): the probability of every 4096-sample chunk"""
    s, out = Stream(), []
    x = np.asarray(audio, np.float32)
    for i in range(0, x.size, CHUNK):
        inp, nxt = model_input(s.context, x[i:i + CHUNK])
        p, s.hidden, s.cell = _one(model, inp, s.hidden, s.cell)
        s.context = nxt
        out.append(p)
    return np.array(out, np.float32)


def segment(probabilities, total_samples, cfg):
    """[(start, end)] sample ranges of segmentSpeech(from:totalSamples:config:)"""
    p = np.ascontiguousarray(probabilities, np.float32).reshape(-1)
    r = _resolved(cfg)
    out = np.zeros(2 * max(1, p.size), np.int64)
    n = lib().oracle_vad_segment(p.ctypes.data, p.size, int(total_samples), C.byref(r), out.ctypes.data, p.size)
    assert n <= p.size
    return [(int(out[2 * k]), int(out[2 * k + 1])) for k in range(n)]


def fsmn_decide(silence):
    """[(startMs, endMs)] of FsmnVadManager.decide(silence:)"""
    s = np.ascontiguousarray(silence, np.float32).reshape(-1)
    cap = (s.size + 1) // 2
    out = np.zeros(2 * max(1, cap), np.int64)
    n = lib().oracle_fsmn_decide(s.ctypes.data, s.size, out.ctypes.data, cap)
    assert n <= cap
    return [(int(out[2 * k]), int(out[2 * k + 1])) for k in range(n)]


class Tick:
    """S sessions carried natively (oracle_vad_tick): one call runs a whole tick, session after session"""

    def __init__(self, S):
        self.S = S
        self.states = np.tile(np.array([0, 0, -1], np.int64), (S, 1))
        self.contexts = np.zeros((S, CONTEXT), np.float32)
        self.hidden = np.zeros((S, STATE), np.float32)
        self.cell = np.zeros((S, STATE), np.float32)
        self.inputs = np.zeros((S, CHUNK + CONTEXT), np.float32)
        self.hidden_out = np.zeros((S, STATE), np.float32)
        self.cell_out = np.zeros((S, STATE), np.float32)
        self.events = np.zeros((S, 2), np.int64)

    def run(self, audio, offsets, probability, new_hidden, new_cell, r):
        """audio and offsets as fa_vad_stream_model_inputs takes them; r a Resolved; events [S x 2] afterwards"""
        a = [np.ascontiguousarray(x, dt) for x, dt in ((audio, np.float32), (offsets, np.int64),
                                                       (probability, np.float32), (new_hidden, np.float32),
                                                       (new_cell, np.float32))]
        lib().oracle_vad_tick(self.S, self.states.ctypes.data, self.contexts.ctypes.data, self.hidden.ctypes.data,
                              self.cell.ctypes.data, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data,
                              a[3].ctypes.data, a[4].ctypes.data, C.byref(r), self.inputs.ctypes.data,
                              self.hidden_out.ctypes.data, self.cell_out.ctypes.data, self.events.ctypes.data)
        return self.events


def segment_batch(probs, offsets, total_samples, r):
    """oracle_vad_segment_batch over packed clips: (counts, pairs [total x 2])"""
    p = np.ascontiguousarray(probs, np.float32)
    off = np.ascontiguousarray(offsets, np.int64)
    ts = np.ascontiguousarray(total_samples, np.int64)
    out = np.zeros((max(1, p.size), 2), np.int64)
    counts = np.zeros(ts.size, np.int64)
    n = lib().oracle_vad_segment_batch(p.ctypes.data, off.ctypes.data, ts.size, ts.ctypes.data, C.byref(r),
                                       out.ctypes.data, counts.ctypes.data)
    return counts, out[:n]
