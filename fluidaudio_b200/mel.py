"""Host-side mirror of ``AudioMelSpectrogram`` (Sources/FluidAudio/Shared/AudioMelSpectrogram.swift:18-121).

Same constructor parameters, same three entry points (``compute`` :132, ``compute_flat`` :185,
``compute_flat_transposed`` :299/:325), same return tuples, same "empty" guards, same non-thread-safety
(one instance per stream of calls).  All arithmetic happens in the sm_90a kernel behind ``fa_mel_*``.
"""
from __future__ import annotations

import ctypes as C
import enum

import numpy as np

from . import _lib


class PaddingMode(enum.IntEnum):
    center = 0        # AudioMelSpectrogram.PaddingMode.center
    pre_padded = 1    # .prePadded


class LogFloorMode(enum.IntEnum):
    additive = 0
    clamped = 1


class Precision(enum.IntEnum):
    f64 = 0           # FA_MEL_PRECISION_F64: transform in FP64, rounded once (default; parity with the oracle ~5e-6)
    f32 = 1           # FA_MEL_PRECISION_F32: float32 transform like vDSP_DFT, two frames per warp


_TIME_MAJOR, _MEL_MAJOR = 0, 1
_LEGACY = 2


class AudioMelSpectrogram:
    def __init__(self, sample_rate: int = 16000, n_mels: int = 128, n_fft: int = 512, hop_length: int = 160,
                 win_length: int = 400, preemph: float = 0.97, pad_to: int = 0, log_floor: float = 2.0 ** -24,
                 log_floor_mode: LogFloorMode = LogFloorMode.additive, window_periodic: bool = False,
                 precision: Precision = Precision.f64):
        self.sample_rate, self.n_mels, self.n_fft = sample_rate, n_mels, n_fft
        self.hop_length, self.win_length, self.preemph = hop_length, win_length, preemph
        self.pad_to = max(1, pad_to)
        self._L = _lib.load()
        cfg = _lib.MelConfig(sample_rate, n_mels, n_fft, hop_length, win_length, preemph, pad_to, log_floor,
                             int(log_floor_mode), int(bool(window_periodic)))
        h = C.c_void_p()
        _lib.check(self._L.fa_mel_create(C.byref(cfg), C.byref(h)), "fa_mel_create")
        self._h = h
        self.precision = Precision(precision)
        if self.precision != Precision.f64:
            self.set_precision(self.precision)

    def set_precision(self, precision: Precision):
        """Not part of the Swift class: selects the transform arithmetic (see include/fluidaudio_b200.h)."""
        _lib.check(self._L.fa_mel_set_precision(self._h, int(precision)), "fa_mel_set_precision")
        self.precision = Precision(precision)

    def close(self):
        if getattr(self, "_h", None) is not None:
            self._L.fa_mel_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- debug getters (:486-493) ---------------------------------------------------------------------------
    def get_hann_window(self) -> np.ndarray:
        out = np.zeros(self.win_length, np.float32)
        _lib.check(self._L.fa_mel_get_window(self._h, out.ctypes.data, out.size), "fa_mel_get_window")
        return out

    def get_filterbank(self) -> np.ndarray:
        out = np.zeros((self.n_mels, self.n_fft // 2 + 1), np.float32)
        _lib.check(self._L.fa_mel_get_filterbank(self._h, out.ctypes.data, out.size), "fa_mel_get_filterbank")
        return out

    def frame_count(self, sample_count: int, padding_mode: int = PaddingMode.center, expected=None) -> int:
        return int(self._L.fa_mel_frame_count(self._h, sample_count, int(padding_mode),
                                              -1 if expected is None else int(expected)))

    # ---- host-buffer entry points ---------------------------------------------------------------------------
    def _run(self, audio, last, mode, expected, layout, out=None):
        audio = np.ascontiguousarray(audio, np.float32)
        n = audio.size
        T = self.frame_count(n, mode, None if mode == _LEGACY else expected)
        empty = T <= 0 or n == 0
        Tp = 1 if empty else (T if mode == _LEGACY else -(-T // self.pad_to) * self.pad_to)
        need = self.n_mels * Tp
        if out is None:
            out = np.empty(need, np.float32)
        elif out.size < need:
            raise ValueError(f"output buffer too small: need {need} floats")
        ml, nf = C.c_int64(), C.c_int64()
        _lib.check(self._L.fa_mel_compute(self._h, _lib.ptr(audio) if n else None, n, float(last), int(mode),
                                          -1 if expected is None else int(expected), layout, out.ctypes.data,
                                          out.size, C.byref(ml), C.byref(nf)), "fa_mel_compute")
        return out, int(ml.value), int(nf.value)

    def compute(self, audio):
        """``compute(audio:)`` → (mel [1, nMels, T], melLength).  No pre-emphasis, no centre padding."""
        out, ml, _ = self._run(audio, 0.0, _LEGACY, None, _MEL_MAJOR)
        if ml == 0:
            return np.zeros((0,), np.float32), 0
        return out[: self.n_mels * ml].reshape(1, self.n_mels, ml), ml

    def compute_flat(self, audio, last_audio_sample: float = 0.0):
        """``computeFlat`` → (mel flat [nMels * numFrames] mel-major, melLength, numFrames)."""
        out, ml, nf = self._run(audio, last_audio_sample, PaddingMode.center, None, _MEL_MAJOR)
        return out[: self.n_mels * nf], ml, nf

    def compute_flat_transposed(self, audio, last_audio_sample: float = 0.0,
                                padding_mode: PaddingMode = PaddingMode.center, expected_frame_count=None, out=None):
        """``computeFlatTransposed`` → (mel flat [numFrames * nMels] time-major, melLength, numFrames)."""
        out, ml, nf = self._run(audio, last_audio_sample, padding_mode, expected_frame_count, _TIME_MAJOR, out)
        return out[: self.n_mels * nf], ml, nf

    # ---- AudioConverter.resample + computeFlatTransposed fused on the device --------------------------------
    def compute_from_pcm(self, pcm, input_rate: float, channels: int | None = None, interleaved: bool = False,
                         last_audio_sample: float = 0.0, padding_mode: PaddingMode = PaddingMode.center,
                         time_major: bool = True, algorithm: int = 0, out=None):
        """PCM (float32 / int16, any channel count and rate) -> log-mel, one call: the raw PCM is the only thing that
        crosses PCIe on the way in, mixdown + resampling to ``sample_rate`` + log-mel run back to back in HBM.
        Returns (mel flat, melLength, numFrames, resampledCount)."""
        from .audio_converter import _as_pcm, _format
        a, frames, channels = _as_pcm(pcm, channels, interleaved)
        fmt = _format(input_rate, self.sample_rate, channels, a.dtype, interleaved, algorithm)
        n = int(self._L.fa_resample_output_count(C.byref(fmt), frames))
        T = self.frame_count(n, padding_mode)
        Tp = 1 if (T <= 0 or n == 0) else -(-T // self.pad_to) * self.pad_to
        need = Tp * self.n_mels
        if out is None:
            out = np.empty(need, np.float32)
        elif out.size < need:
            raise ValueError(f"output buffer too small: need {need} floats")
        ml, nf, rs = C.c_int64(), C.c_int64(), C.c_int64()
        _lib.check(self._L.fa_audio_to_mel(self._h, a.ctypes.data if a.size else None, frames, C.byref(fmt),
                                           float(last_audio_sample), int(padding_mode), 0 if time_major else 1,
                                           out.ctypes.data, out.size, C.byref(ml), C.byref(nf), C.byref(rs)),
                   "fa_audio_to_mel")
        return out[: self.n_mels * nf.value], int(ml.value), int(nf.value), int(rs.value)

    # ---- batch of independent clips (BASELINE config 4) -------------------------------------------------------
    def compute_batch(self, clips, last_samples=None, padding_mode: PaddingMode = PaddingMode.center,
                      time_major: bool = True, packed_audio=None, offsets=None, out=None):
        """``clips``: list of float32 arrays (or pass ``packed_audio`` + ``offsets``).  Returns
        (out flat float32, out_offsets int64 [count+1], mel_lengths int64, num_frames int64)."""
        if packed_audio is None:
            clips = [np.ascontiguousarray(c, np.float32).reshape(-1) for c in clips]
            offsets = np.zeros(len(clips) + 1, np.int64)
            offsets[1:] = np.cumsum([c.size for c in clips])
            packed_audio = np.concatenate(clips) if clips else np.zeros(0, np.float32)
        offsets = np.ascontiguousarray(offsets, np.int64)
        count = offsets.size - 1
        out_offsets = np.zeros(count + 1, np.int64)
        for i in range(count):
            n = int(offsets[i + 1] - offsets[i])
            T = self.frame_count(n, padding_mode)
            Tp = 1 if (T <= 0 or n == 0) else -(-T // self.pad_to) * self.pad_to
            out_offsets[i + 1] = out_offsets[i] + Tp * self.n_mels
        if out is None:
            out = np.empty(int(out_offsets[-1]), np.float32)
        ml = np.zeros(count, np.int64)
        nf = np.zeros(count, np.int64)
        last = None if last_samples is None else np.ascontiguousarray(last_samples, np.float32)
        _lib.check(self._L.fa_mel_compute_batch(self._h, packed_audio.ctypes.data, offsets.ctypes.data, count,
                                                _lib.ptr(last), int(padding_mode), 0 if time_major else 1,
                                                out.ctypes.data, out_offsets.ctypes.data, ml.ctypes.data,
                                                nf.ctypes.data), "fa_mel_compute_batch")
        return out, out_offsets, ml, nf

    # ---- device-resident entry point (kernel-only timing, pipelines that keep audio in HBM) -------------------
    def compute_device(self, d_audio: "_lib.DeviceBuffer", sample_count: int, d_out: "_lib.DeviceBuffer",
                       last_audio_sample: float = 0.0, padding_mode: PaddingMode = PaddingMode.center,
                       expected_frame_count=None, time_major: bool = True):
        ml, nf = C.c_int64(), C.c_int64()
        _lib.check(self._L.fa_mel_compute_device(self._h, d_audio.ptr, sample_count, float(last_audio_sample),
                                                 int(padding_mode),
                                                 -1 if expected_frame_count is None else int(expected_frame_count),
                                                 0 if time_major else 1, d_out.ptr, d_out.nbytes // 4,
                                                 C.byref(ml), C.byref(nf)), "fa_mel_compute_device")
        return int(ml.value), int(nf.value)

    def timer_start(self):
        _lib.check(self._L.fa_mel_timer_start(self._h), "fa_mel_timer_start")

    def timer_stop_ms(self) -> float:
        ms = C.c_float()
        _lib.check(self._L.fa_mel_timer_stop_ms(self._h, C.byref(ms)), "fa_mel_timer_stop_ms")
        return float(ms.value)

    def compute_batch_device(self, d_audio, offsets, d_out, out_offsets, padding_mode=PaddingMode.center,
                             time_major: bool = True):
        offsets = np.ascontiguousarray(offsets, np.int64)
        out_offsets = np.ascontiguousarray(out_offsets, np.int64)
        count = offsets.size - 1
        ml = np.zeros(count, np.int64)
        nf = np.zeros(count, np.int64)
        _lib.check(self._L.fa_mel_compute_batch_device(self._h, d_audio.ptr, offsets.ctypes.data, count, None,
                                                       int(padding_mode), 0 if time_major else 1, d_out.ptr,
                                                       out_offsets.ctypes.data, ml.ctypes.data, nf.ctypes.data),
                   "fa_mel_compute_batch_device")
        return ml, nf


class MelStreams:
    """Live log-mel streams on one ``AudioMelSpectrogram``: SortformerDiarizer's incremental mel stream
    (Diarizer/Sortformer/SortformerDiarizer.swift:204-217, :417-424, :842-901) for any number of sessions, each push
    advancing every session it names with a fixed number of launches (``fa_mel_stream_*``).  The sessions share the
    handle's configuration (``pad_to`` 0 or 1, ``hop_length <= win_length``) and precision."""

    def __init__(self, mel: AudioMelSpectrogram):
        self.mel = mel
        self.n_mels = mel.n_mels
        self._L = mel._L

    def open(self) -> int:
        """resetMelStreamLocked: a new session (the lowest free id) with nFFT/2 zeros buffered."""
        sid = C.c_int32()
        _lib.check(self._L.fa_mel_stream_open(self.mel._h, C.byref(sid)), "fa_mel_stream_open")
        return int(sid.value)

    def close(self, session: int):
        _lib.check(self._L.fa_mel_stream_close(self.mel._h, int(session)), "fa_mel_stream_close")

    def pending_frames(self, session: int, n: int, finish: bool = False) -> int:
        """Rows the next push of ``n`` samples (and ``finish``) to ``session`` emits."""
        v = int(self._L.fa_mel_stream_frames(self.mel._h, int(session), int(n), int(bool(finish))))
        if v < 0:
            raise ValueError(f"session {session} is not open (or n < 0)")
        return v

    def _pack(self, chunks, finish):
        chunks = {int(s): a for s, a in chunks.items()}
        done = {int(f) for f in finish}
        ids = list(chunks) + sorted(done - set(chunks))
        arrays = [np.ascontiguousarray(chunks.get(s, np.zeros(0, np.float32)), np.float32).reshape(-1) for s in ids]
        offsets = np.zeros(len(ids) + 1, np.int64)
        offsets[1:] = np.cumsum([a.size for a in arrays])
        audio = np.concatenate(arrays) if arrays else np.zeros(0, np.float32)
        fin = np.array([1 if s in done else 0 for s in ids], np.int32)
        return np.array(ids, np.int32), audio, offsets, fin

    def push(self, chunks: dict, finish=()) -> dict:
        """``chunks``: {session: samples} (addAudio); sessions in ``finish`` are finalised after their samples
        (padAndEmitRemainingMelLocked).  Returns {session: [frames x nMels] float32} for every session named."""
        ids, audio, offsets, fin = self._pack(chunks, finish)
        counts = [self.pending_frames(s, int(offsets[i + 1] - offsets[i]), bool(fin[i])) for i, s in enumerate(ids)]
        out = np.empty(max(1, sum(counts)) * self.n_mels, np.float32)
        frames = np.zeros(ids.size, np.int64)
        _lib.check(self._L.fa_mel_stream_push(self.mel._h, ids.size, _lib.ptr(ids), _lib.ptr(audio) if audio.size else None,
                                              _lib.ptr(offsets), _lib.ptr(fin), out.ctypes.data, out.size,
                                              frames.ctypes.data), "fa_mel_stream_push")
        res, row = {}, 0
        for s, f in zip(ids.tolist(), frames.tolist()):
            res[s] = out[row * self.n_mels:(row + f) * self.n_mels].reshape(f, self.n_mels)
            row += f
        return res

    def push_device(self, sessions, d_audio: "_lib.DeviceBuffer", offsets, d_out: "_lib.DeviceBuffer", finish=None,
                    out_offset: int = 0) -> np.ndarray:
        """The push with samples and rows in HBM: session ``sessions[i]`` reads ``d_audio[offsets[i]:offsets[i+1]]``; the
        rows land at float ``out_offset`` of ``d_out`` in call order.  Asynchronous; returns the frame counts."""
        ids = np.ascontiguousarray(sessions, np.int32)
        offsets = np.ascontiguousarray(offsets, np.int64)
        fin = None if finish is None else np.ascontiguousarray(finish, np.int32)
        frames = np.zeros(ids.size, np.int64)
        out_ptr = d_out.ptr.value + 4 * int(out_offset)
        _lib.check(self._L.fa_mel_stream_push_device(self.mel._h, ids.size, _lib.ptr(ids), d_audio.ptr, _lib.ptr(offsets),
                                                     _lib.ptr(fin), out_ptr, d_out.nbytes // 4 - int(out_offset),
                                                     frames.ctypes.data), "fa_mel_stream_push_device")
        return frames


def normalize_per_feature(mel_time_major: np.ndarray, valid_frames: int) -> np.ndarray:
    """UnifiedMelExtractor.normalizePerFeature (UnifiedMelExtractor.swift:88-113) on a [frames x nMels] array."""
    x = np.ascontiguousarray(mel_time_major, np.float32).copy()
    _lib.check(_lib.load().fa_mel_normalize_per_feature(x.ctypes.data, x.shape[0], x.shape[1], int(valid_frames)),
               "fa_mel_normalize_per_feature")
    return x


def to_channel_major(mel_time_major: np.ndarray) -> np.ndarray:
    """NemotronMelExtractor.melSpectrogram's [T x M] → [1, M, T] re-layout (NemotronMelExtractor.swift:44-67)."""
    return np.ascontiguousarray(mel_time_major.T)[None]


class UnifiedMelExtractor:
    """ASR/Parakeet/Unified/UnifiedMelExtractor.swift:15-113: NeMo `AudioToMelSpectrogramPreprocessor` features with
    `normalize: per_feature`, packed for the encoder.  The normalisation and the [1, nMels, T] packing run on the GPU
    behind the mel kernel (`fa_mel_unified_features`)."""

    def __init__(self, window_samples: int, n_mels: int = 128):
        self.window_samples = int(window_samples)
        self.n_mels = n_mels
        self.hop_length = 160
        self.total_frames = self.window_samples // self.hop_length + 1
        self._mel = AudioMelSpectrogram(sample_rate=16000, n_mels=n_mels, n_fft=512, hop_length=160, win_length=400,
                                        preemph=0.97, pad_to=0, window_periodic=False)

    def features(self, window: np.ndarray, valid_count: int) -> tuple[np.ndarray, np.ndarray]:
        """Returns (mel [1, nMels, totalFrames] float32, length [1] int32) — the CoreML preprocessor's contract."""
        window = np.ascontiguousarray(window, np.float32)
        if window.size != self.window_samples:
            raise ValueError(f"window must hold {self.window_samples} samples, got {window.size}")
        out = np.zeros((1, self.n_mels, self.total_frames), np.float32)
        T, valid = C.c_int64(), C.c_int32()
        _lib.check(self._mel._L.fa_mel_unified_features(self._mel._h, window.ctypes.data, window.size, int(valid_count),
                                                        out.ctypes.data, out.size, C.byref(T), C.byref(valid)),
                   "fa_mel_unified_features")
        assert T.value == self.total_frames
        return out, np.array([valid.value], np.int32)


class LSEENDMelFrontend:
    """The mel half of LSEENDPreprocessor (Diarizer/LS-EEND/LSEENDPreprocessor.swift:70-81, 249-283): `.prePadded`
    log-mel with preemph 0 / periodic Hann / clamped floor 1e-10, log10 scaling, cumulative mean normalisation whose
    state (`cmn_mean`, `cmn_count`) lives here exactly as in the preprocessor; `reset()` as :236-245."""

    def __init__(self, n_mels: int = 23, n_fft: int = 512, hop_length: int = 160, win_length: int = 400,
                 sample_rate: int = 16000):
        self.n_mels = n_mels
        self._mel = AudioMelSpectrogram(sample_rate=sample_rate, n_mels=n_mels, n_fft=n_fft, hop_length=hop_length,
                                        win_length=win_length, preemph=0.0, pad_to=0, log_floor=1e-10,
                                        log_floor_mode=LogFloorMode.clamped, window_periodic=True)
        self.reset()

    def reset(self):
        self.cmn_mean = np.zeros(self.n_mels, np.float32)
        self.cmn_count = 0

    def process(self, audio_chunk: np.ndarray) -> np.ndarray:
        """One popped audio chunk (already carrying its left / right context) -> [frames x nMels] features."""
        chunk = np.ascontiguousarray(audio_chunk, np.float32)
        T = self._mel.frame_count(chunk.size, PaddingMode.pre_padded)
        out = np.zeros((max(T, 0), self.n_mels), np.float32)
        cnt, frames = C.c_int64(self.cmn_count), C.c_int64()
        _lib.check(self._mel._L.fa_mel_lseend_features(self._mel._h, chunk.ctypes.data, chunk.size,
                                                       self.cmn_mean.ctypes.data, C.byref(cnt), out.ctypes.data,
                                                       out.size, C.byref(frames)), "fa_mel_lseend_features")
        self.cmn_count = cnt.value
        return out[: frames.value]
