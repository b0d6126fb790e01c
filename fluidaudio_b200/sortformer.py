"""Sortformer's streaming state on the GPU (``fa_sortformer_*``): SortformerStateUpdater.streamingUpdate
(Diarizer/Sortformer/SortformerStateUpdater.swift) for many live sessions, each a SortformerStreamingState
(SortformerTypes.swift:270-327) in HBM, and the next model call's padded inputs (SortformerModelInference.swift:266-303).

The model itself runs outside the library; a deployment loops ``model_inputs`` -> model -> ``update`` per chunk tick,
with every session of the tick in one call.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, fields
from types import SimpleNamespace

import numpy as np

from . import _lib

D, S = 512, 4   # preEncoderDims, numSpeakers
PRESETS = ("default", "fastV2", "fastV2_1", "balancedV2", "balancedV2_1", "highContextV2", "highContextV2_1",
           "efficientV2_1")


@dataclass
class SortformerConfig:
    """The `var` fields of SortformerConfig (SortformerTypes.swift:31-97); defaults are the init's."""
    chunk_len: int = 6
    chunk_left_context: int = 1
    chunk_right_context: int = 7
    fifo_len: int = 40
    spkcache_len: int = 188
    spkcache_update_period: int = 31
    spkcache_sil_frames_per_spk: int = 3
    silence_threshold: float = 0.2
    pred_score_threshold: float = 0.25
    scores_boost_latest: float = 0.05
    strong_boost_rate: float = 0.75
    weak_boost_rate: float = 1.5
    min_pos_scores_rate: float = 0.5

    @classmethod
    def preset(cls, name: str = "default") -> "SortformerConfig":
        """One of the reference's static configs (``PRESETS``)."""
        c = _lib.SortformerConfig()
        _lib.check(_lib.load().fa_sortformer_default_config(C.byref(c), PRESETS.index(name)), "fa_sortformer_default_config")
        return cls._from_c(c)

    @classmethod
    def _from_c(cls, c) -> "SortformerConfig":
        return cls(**{f.name: getattr(c, f.name) for f in fields(cls)})

    def to_c(self) -> "_lib.SortformerConfig":
        return _lib.SortformerConfig(**{f.name: getattr(self, f.name) for f in fields(self)})

    def resolved(self, max_core_frames: int = 0):
        """(the configuration after the init's clamps, max_core) as fa_sortformer_create applies them"""
        out, mc = _lib.SortformerConfig(), C.c_int32()
        _lib.check(_lib.load().fa_sortformer_resolve_config(C.byref(self.to_c()), int(max_core_frames), C.byref(out),
                                                            C.byref(mc)), "fa_sortformer_resolve_config")
        return SortformerConfig._from_c(out), int(mc.value)


def step_lengths(cfg: SortformerConfig, spkcache_length: int, fifo_length: int, has_spkcache_preds: bool,
                 emb_length: int, pred_rows: int, left_context: int, right_context: int, max_core_frames: int = 0):
    """The host plan of one streamingUpdate (fa_sortformer_step): namespace(core, pop, compress, spkcache_length,
    fifo_length, has_spkcache_preds) after it; raises FluidAudioError(INVALID_ARGUMENT) where the reference throws."""
    lin = np.array([spkcache_length, fifo_length, int(bool(has_spkcache_preds))], np.int32)
    out = np.zeros(6, np.int32)
    _lib.check(_lib.load().fa_sortformer_step(C.byref(cfg.to_c()), int(max_core_frames), lin.ctypes.data, int(emb_length),
                                              int(pred_rows), int(left_context), int(right_context), out.ctypes.data),
               "fa_sortformer_step")
    return SimpleNamespace(core=int(out[0]), pop=int(out[1]), compress=bool(out[2]), spkcache_length=int(out[3]),
                           fifo_length=int(out[4]), has_spkcache_preds=bool(out[5]))


class SortformerStreams:
    """Sessions of Sortformer streaming state on the current device.  ``max_core_frames`` (0: chunkLen) bounds the core
    frames of one update.  Not thread-safe, like the reference's state."""

    def __init__(self, cfg: SortformerConfig | None = None, max_core_frames: int = 0):
        self._L = _lib.load()
        self.config, self.max_core = (cfg or SortformerConfig()).resolved(max_core_frames)
        h = C.c_void_p()
        _lib.check(self._L.fa_sortformer_create(C.byref(self.config.to_c()), self.max_core, C.byref(h)),
                   "fa_sortformer_create")
        self._h = h

    def close_handle(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._L.fa_sortformer_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close_handle()
        except Exception:
            pass

    def open(self) -> int:
        """A fresh SortformerStreamingState (the lowest free id)."""
        sid = C.c_int32()
        _lib.check(self._L.fa_sortformer_open(self._h, C.byref(sid)), "fa_sortformer_open")
        return int(sid.value)

    def close(self, session: int):
        _lib.check(self._L.fa_sortformer_close(self._h, int(session)), "fa_sortformer_close")

    @staticmethod
    def _ints(a, n):
        return None if a is None else np.ascontiguousarray(np.broadcast_to(np.asarray(a, np.int32), (n,)))

    def update(self, sessions, chunk_embs, preds, emb_lengths=None, left_context=None, right_context=None):
        """streamingUpdate for session ``sessions[i]`` with batch row i of ``chunk_embs`` [n x rows x 512] and ``preds``
        [n x pred_rows x 4].  ``emb_lengths`` defaults to all rows; a context of None is the streaming rule
        (SortformerDiarizer.swift:553-554).  Returns ([confirmed [core x 4]], [tentative [rc x 4]]) per session."""
        ids = np.ascontiguousarray(sessions, np.int32).reshape(-1)
        n = ids.size
        e = np.ascontiguousarray(chunk_embs, np.float32)
        p = np.ascontiguousarray(preds, np.float32)
        e = e.reshape(n, e.size // (n * D) if n else 0, D)
        p = p.reshape(n, p.size // (n * S) if n else 0, S)
        el = self._ints(e.shape[1] if emb_lengths is None else emb_lengths, n)
        lc, rc = self._ints(left_context, n), self._ints(right_context, n)
        cap = max(1, n * max(e.shape[1], 1) * S)
        conf, tent = np.empty(cap, np.float32), np.empty(cap, np.float32)
        cr, tr = np.zeros(n, np.int64), np.zeros(n, np.int64)
        _lib.check(self._L.fa_sortformer_update(self._h, n, _lib.ptr(ids), e.ctypes.data, e.shape[1], p.ctypes.data,
                                                p.shape[1], _lib.ptr(el), _lib.ptr(lc), _lib.ptr(rc), conf.ctypes.data,
                                                cap, tent.ctypes.data, cap, cr.ctypes.data, tr.ctypes.data),
                   "fa_sortformer_update")
        return self._split(conf, cr), self._split(tent, tr)

    @staticmethod
    def _split(buf, rows):
        out, r = [], 0
        for k in rows.tolist():
            out.append(buf[r * S:(r + k) * S].reshape(k, S).copy())
            r += k
        return out

    def update_device(self, sessions, d_embs: "_lib.DeviceBuffer", emb_rows: int, d_preds: "_lib.DeviceBuffer",
                      pred_rows: int, d_confirmed: "_lib.DeviceBuffer", d_tentative: "_lib.DeviceBuffer",
                      emb_lengths=None, left_context=None, right_context=None):
        """The update on HBM buffers, asynchronous on the handle's stream; returns (confirmed_rows, tentative_rows)."""
        ids = np.ascontiguousarray(sessions, np.int32).reshape(-1)
        n = ids.size
        el = self._ints(emb_rows if emb_lengths is None else emb_lengths, n)
        lc, rc = self._ints(left_context, n), self._ints(right_context, n)
        cr, tr = np.zeros(n, np.int64), np.zeros(n, np.int64)
        _lib.check(self._L.fa_sortformer_update_device(self._h, n, _lib.ptr(ids), d_embs.ptr, int(emb_rows), d_preds.ptr,
                                                       int(pred_rows), _lib.ptr(el), _lib.ptr(lc), _lib.ptr(rc),
                                                       d_confirmed.ptr, d_confirmed.nbytes // 4, d_tentative.ptr,
                                                       d_tentative.nbytes // 4, cr.ctypes.data, tr.ctypes.data),
                   "fa_sortformer_update_device")
        return cr, tr

    def model_inputs(self, sessions):
        """(spkcache [n x spkcacheLen x 512], fifo [n x fifoLen x 512], spkcache_lengths [n], fifo_lengths [n])"""
        ids = np.ascontiguousarray(sessions, np.int32).reshape(-1)
        n = ids.size
        sc = np.empty((n, self.config.spkcache_len, D), np.float32)
        ff = np.empty((n, self.config.fifo_len, D), np.float32)
        sl, fl = np.zeros(n, np.int32), np.zeros(n, np.int32)
        _lib.check(self._L.fa_sortformer_model_inputs(self._h, n, _lib.ptr(ids), sc.ctypes.data, ff.ctypes.data,
                                                      sl.ctypes.data, fl.ctypes.data), "fa_sortformer_model_inputs")
        return sc, ff, sl, fl

    def model_inputs_device(self, sessions, d_spkcache: "_lib.DeviceBuffer", d_fifo: "_lib.DeviceBuffer"):
        """The model inputs written to HBM (asynchronous); returns (spkcache_lengths, fifo_lengths)."""
        ids = np.ascontiguousarray(sessions, np.int32).reshape(-1)
        sl, fl = np.zeros(ids.size, np.int32), np.zeros(ids.size, np.int32)
        _lib.check(self._L.fa_sortformer_model_inputs_device(self._h, ids.size, _lib.ptr(ids), d_spkcache.ptr, d_fifo.ptr,
                                                             sl.ctypes.data, fl.ctypes.data),
                   "fa_sortformer_model_inputs_device")
        return sl, fl

    def state(self, session: int):
        """The session's full state: namespace(spkcache, spkcache_preds (None when absent), fifo, fifo_preds (None when
        absent), mean_silence, silence_frames, spkcache_length, fifo_length, chunks)."""
        c = self.config
        sc, sp = np.zeros((c.spkcache_len, D), np.float32), np.zeros((c.spkcache_len, S), np.float32)
        ff, fp = np.zeros((c.fifo_len, D), np.float32), np.zeros((c.fifo_len, S), np.float32)
        mean, info = np.zeros(D, np.float32), _lib.SortformerSessionInfo()
        _lib.check(self._L.fa_sortformer_session_state(self._h, int(session), C.byref(info), sc.ctypes.data, sp.ctypes.data,
                                                       ff.ctypes.data, fp.ctypes.data, mean.ctypes.data),
                   "fa_sortformer_session_state")
        n, m = info.spkcache_length, info.fifo_length
        return SimpleNamespace(spkcache=sc[:n], spkcache_preds=sp[:n] if info.has_spkcache_preds else None, fifo=ff[:m],
                               fifo_preds=fp[:m] if info.has_fifo_preds else None, mean_silence=mean,
                               silence_frames=int(info.silence_frames), spkcache_length=n, fifo_length=m,
                               has_spkcache_preds=bool(info.has_spkcache_preds), has_fifo_preds=bool(info.has_fifo_preds),
                               chunks=int(info.chunks))
