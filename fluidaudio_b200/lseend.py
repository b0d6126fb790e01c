"""LS-EEND live feature streams on the GPU (``fa_lseend_stream_*``): LSEENDFeatureProvider
(Diarizer/LS-EEND/LSEENDPreprocessor.swift:46-384) for many live sessions, from audio at the model's rate to the model's
input chunks: the audio queue, the log10 log-mel, the running mean normalisation, the mel queue, the decoder mask and
the warm-up counts.

``LSEENDFeatureStreams`` owns the sessions in HBM; one ``push`` advances every session of a tick and returns every chunk
it made ready.  ``LSEENDFeatureProvider`` is one session seen as the reference's class: ``enqueue_audio``,
``ready_chunks``, ``emit_next_chunk``, ``drain_right_context_with_silence``, ``take_snapshot``, ``rollback`` and
``reset``.  The LS-EEND model and its recurrent state are the caller's.
"""
from __future__ import annotations

import ctypes as C
from collections import deque
from dataclasses import dataclass, fields
from types import SimpleNamespace

import numpy as np

from . import _lib
from .mel import Precision


@dataclass
class LSEENDStreamConfig:
    """The LSEENDMetadata fields the provider reads (LSEENDTypes.swift:10-58) and the transform precision."""
    sample_rate: int = 16000
    n_mels: int = 23
    hop_length: int = 160
    win_length: int = 400
    context_size: int = 7
    subsampling: int = 10
    chunk_size: int = 1
    conv_delay: int = 2
    precision: int = int(Precision.f64)

    def _c(self) -> _lib.LSEENDStreamConfig:
        return _lib.LSEENDStreamConfig(*(int(getattr(self, f.name)) for f in fields(self)))

    def resolve(self) -> SimpleNamespace:
        """The sizes the provider's init derives (n_fft, mel_frames, chunk_samples, flush_samples, ...); no device."""
        s = _lib.LSEENDStreamSizes()
        _lib.check(_lib.load().fa_lseend_stream_resolve(C.byref(self._c()), C.byref(s)), "fa_lseend_stream_resolve")
        return SimpleNamespace(**{k: int(getattr(s, k)) for k, _ in s._fields_})


class LSEENDFeatureStreams:
    """Many live LS-EEND feature providers in HBM on one handle: they share its configuration and stream."""

    def __init__(self, config: LSEENDStreamConfig):
        self.config = config
        self.sizes = config.resolve()
        self.n_mels = int(config.n_mels)
        self._L = _lib.load()
        h = C.c_void_p()
        _lib.check(self._L.fa_lseend_stream_create(C.byref(config._c()), C.byref(h)), "fa_lseend_stream_create")
        self._h = h

    def close_handle(self):
        if getattr(self, "_h", None):
            self._L.fa_lseend_stream_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close_handle()
        except Exception:
            pass

    def open(self) -> int:
        """A fresh provider (the lowest free id)."""
        sid = C.c_int32()
        _lib.check(self._L.fa_lseend_stream_open(self._h, C.byref(sid)), "fa_lseend_stream_open")
        return int(sid.value)

    def close(self, session: int):
        _lib.check(self._L.fa_lseend_stream_close(self._h, int(session)), "fa_lseend_stream_close")

    def chunks(self, session: int, n: int, drain: bool = False) -> int:
        """Chunks the next push of ``n`` samples (and the drain) to ``session`` emits."""
        v = int(self._L.fa_lseend_stream_chunks(self._h, int(session), int(n), int(bool(drain))))
        if v < 0:
            raise ValueError(f"session {session} is not open (or n is outside 0 .. 2^40)")
        return v

    def push(self, chunks: dict, drain=()):
        """``chunks``: {session: samples}; sessions in ``drain`` are drained with silence after their samples.  Returns
        {session: (features [k x mel_frames x n_mels], masks [k x chunk_size], warmup [k] int32)} for every session
        named, k its chunks."""
        chunks = {int(s): a for s, a in chunks.items()}
        done = {int(d) for d in drain}
        ids = np.array(list(chunks) + sorted(done - set(chunks)), np.int32)
        arrays = [np.ascontiguousarray(chunks.get(int(s), np.zeros(0, np.float32)), np.float32).reshape(-1) for s in ids]
        offsets = np.zeros(ids.size + 1, np.int64)
        offsets[1:] = np.cumsum([a.size for a in arrays])
        audio = np.concatenate(arrays) if arrays else np.zeros(0, np.float32)
        dr = np.array([1 if int(s) in done else 0 for s in ids], np.int32)
        k = sum(self.chunks(int(s), a.size, bool(d)) for s, a, d in zip(ids, arrays, dr))
        F, T = self.sizes.mel_frames, self.config.chunk_size
        feats = np.empty((max(k, 1), F, self.n_mels), np.float32)
        masks = np.empty((max(k, 1), T), np.float32)
        warm = np.empty(max(k, 1), np.int32)
        counts = np.zeros(ids.size, np.int64)
        _lib.check(self._L.fa_lseend_stream_push(self._h, ids.size, _lib.ptr(ids), _lib.ptr(audio) if audio.size else None,
                                                 _lib.ptr(offsets), _lib.ptr(dr), feats.ctypes.data, feats.size,
                                                 masks.ctypes.data, masks.size, warm.ctypes.data, warm.size,
                                                 counts.ctypes.data), "fa_lseend_stream_push")
        res, c = {}, 0
        for s, n in zip(ids.tolist(), counts.tolist()):
            res[s] = (feats[c:c + n], masks[c:c + n], warm[c:c + n])
            c += n
        return res

    def push_device(self, sessions, d_audio: "_lib.DeviceBuffer", offsets, d_features: "_lib.DeviceBuffer",
                    d_masks: "_lib.DeviceBuffer", d_warmup: "_lib.DeviceBuffer", drain=None) -> np.ndarray:
        """The push with samples and outputs in HBM, asynchronous; returns the chunk counts."""
        ids = np.ascontiguousarray(sessions, np.int32)
        offsets = np.ascontiguousarray(offsets, np.int64)
        dr = None if drain is None else np.ascontiguousarray(drain, np.int32)
        counts = np.zeros(ids.size, np.int64)
        _lib.check(self._L.fa_lseend_stream_push_device(self._h, ids.size, _lib.ptr(ids), d_audio.ptr, _lib.ptr(offsets),
                                                        _lib.ptr(dr), d_features.ptr, d_features.nbytes // 4,
                                                        d_masks.ptr, d_masks.nbytes // 4, d_warmup.ptr,
                                                        d_warmup.nbytes // 4, counts.ctypes.data),
                   "fa_lseend_stream_push_device")
        return counts

    def _each(self, name, sessions):
        ids = np.ascontiguousarray(np.atleast_1d(sessions), np.int32)
        _lib.check(getattr(self._L, name)(self._h, ids.size, _lib.ptr(ids)), name)

    def snapshot(self, sessions):
        """takeSnapshot for each session (one launch)."""
        self._each("fa_lseend_stream_snapshot", sessions)

    def rollback(self, sessions):
        """rollback(to:) each session's snapshot (one launch); the snapshot stays."""
        self._each("fa_lseend_stream_rollback", sessions)

    def reset(self, sessions):
        """reset(): each session fresh (one launch)."""
        self._each("fa_lseend_stream_reset", sessions)

    def state(self, session: int) -> SimpleNamespace:
        """audio [unread samples], mel [unread rows x n_mels], cmn_mean, cmn_count, decoder_mask_end, has_snapshot."""
        info = _lib.LSEENDSessionInfo()
        _lib.check(self._L.fa_lseend_stream_session_state(self._h, int(session), C.byref(info), None, None, None),
                   "fa_lseend_stream_session_state")
        audio = np.zeros(info.audio_samples, np.float32)
        mel = np.zeros((info.mel_rows, self.n_mels), np.float32)
        mean = np.zeros(self.n_mels, np.float32)
        _lib.check(self._L.fa_lseend_stream_session_state(self._h, int(session), C.byref(info), audio.ctypes.data,
                                                          mel.ctypes.data, mean.ctypes.data),
                   "fa_lseend_stream_session_state")
        return SimpleNamespace(audio=audio, mel=mel, cmn_mean=mean, cmn_count=int(info.cmn_count),
                               decoder_mask_end=int(info.decoder_mask_end), has_snapshot=bool(info.has_snapshot))


class LSEENDFeatureProvider:
    """One session as the reference's LSEENDFeatureProvider.  Every push emits what it makes ready, so the chunks wait
    here on the host until ``emit_next_chunk`` takes them; a snapshot keeps them too."""

    def __init__(self, config: LSEENDStreamConfig | None = None, streams: LSEENDFeatureStreams | None = None):
        self.streams = streams if streams is not None else LSEENDFeatureStreams(config or LSEENDStreamConfig())
        self.session = self.streams.open()
        self._ready = deque()
        self._snapshot = None

    def _push(self, samples, drain):
        a = np.ascontiguousarray(samples, np.float32).reshape(-1)
        f, m, w = self.streams.push({self.session: a}, drain=(self.session,) if drain else ())[self.session]
        self._ready.extend((f[i], m[i], int(w[i])) for i in range(len(w)))

    def enqueue_audio(self, samples):
        """enqueueAudio (eager processing), samples at the model's rate."""
        self._push(samples, False)

    def drain_right_context_with_silence(self):
        """drainRightContextWithSilence(flush: true)"""
        self._push(np.zeros(0, np.float32), True)

    @property
    def ready_chunks(self) -> int:
        return len(self._ready)

    def emit_next_chunk(self):
        """(features [mel_frames x n_mels], decoder mask [chunk_size], warm-up frames), or None."""
        return self._ready.popleft() if self._ready else None

    def take_snapshot(self):
        self.streams.snapshot(self.session)
        self._snapshot = list(self._ready)

    def rollback(self):
        if self._snapshot is None:
            raise ValueError("no snapshot taken")
        self.streams.rollback(self.session)
        self._ready = deque(self._snapshot)

    def reset(self):
        self.streams.reset(self.session)
        self._ready.clear()
