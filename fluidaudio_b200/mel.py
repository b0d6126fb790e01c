"""Host-side mirror of ``AudioMelSpectrogram`` (Sources/FluidAudio/Shared/AudioMelSpectrogram.swift:18-121).

Same constructor parameters, same three entry points (``compute`` :132, ``compute_flat`` :185,
``compute_flat_transposed`` :299/:325), same return tuples, same "empty" guards, same non-thread-safety
(one instance per stream of calls).  All arithmetic happens in the sm_90a kernel behind ``fa_mel_*``.
"""
from __future__ import annotations

import ctypes as C
import enum
from dataclasses import dataclass
from typing import NamedTuple

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


class MelFilterbank(enum.IntEnum):   # FA_MEL_FB_*: whose table construction a handle restates
    audio_mel = 0
    cohere = 1
    styletts2 = 2
    luxtts = 3


class CenterEdge(enum.IntEnum):      # FA_MEL_EDGE_*: what .center pads with
    zero = 0
    reflect = 1


_TIME_MAJOR, _MEL_MAJOR = 0, 1
_EX_FIELDS = {name for name, _ in _lib.MelExConfig._fields_} - {"base"}


def ex_config(preset: str | None = None, **fields) -> "_lib.MelExConfig":
    """An ``fa_mel_ex_config``: neutral (``fa_mel_ex_default_config``) or one of the presets ``"cohere"``,
    ``"styletts2"``, ``"luxtts"``, then ``fields`` set by name (base fields such as ``n_mels`` or ex fields such as
    ``spectrum_power``)."""
    L = _lib.load()
    cfg = _lib.MelExConfig()
    init = {None: L.fa_mel_ex_default_config, "cohere": L.fa_mel_preset_cohere, "styletts2": L.fa_mel_preset_styletts2,
            "luxtts": L.fa_mel_preset_luxtts}[preset]
    init(C.byref(cfg))
    for k, v in fields.items():
        setattr(cfg if k in _EX_FIELDS else cfg.base, k, v)
    return cfg
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

    @classmethod
    def from_ex_config(cls, cfg: "_lib.MelExConfig", precision: Precision = Precision.f64) -> "AudioMelSpectrogram":
        """A handle made by ``fa_mel_create_ex``: every method of this class works on it unchanged."""
        self = cls.__new__(cls)
        b = cfg.base
        self.sample_rate, self.n_mels, self.n_fft = b.sample_rate, b.n_mels, b.n_fft
        self.hop_length, self.win_length, self.preemph = b.hop_length, b.win_length, b.preemph
        self.pad_to = max(1, b.pad_to)
        self._L = _lib.load()
        h = C.c_void_p()
        _lib.check(self._L.fa_mel_create_ex(C.byref(cfg), C.byref(h)), "fa_mel_create_ex")
        self._h = h
        self.precision = Precision.f64
        if Precision(precision) != Precision.f64:
            self.set_precision(precision)
        return self

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


# ================================================================================================ torch-style frontends
class CohereMelSpectrogram:
    """ASR/Cohere/CoherePipeline.swift:41-324: NeMo FilterbankFeatures-compatible log-mel (Slaney table over
    ``f_min`` .. ``f_max``, ``|X|^magPower``, additive log guard), per-feature CMVN over the valid frames and
    ``padOrTruncate``.  The STFT, the table product and the log run in the mel kernel, the CMVN and the packing in one
    epilogue kernel behind it (``fa_mel_cohere_features``).  Pre-emphasis is one fused multiply-add per sample where the
    Swift rounds twice (DESIGN §4.1b)."""

    @dataclass(frozen=True)
    class Config:
        sample_rate: int = 16_000
        win_length: int = 400
        hop_length: int = 160
        n_mels: int = 128
        f_min: float = 0.0
        f_max: float = 8_000.0
        preemph: float = 0.97
        mag_power: float = 2.0
        log_zero_guard: float = 5.9604645e-08   # 2^-24
        cmvn_epsilon: float = 1.0e-5

    class Output(NamedTuple):
        mel: np.ndarray          # [nMels x nFrames]
        valid_frames: int

    def __init__(self, config: "CohereMelSpectrogram.Config | None" = None,
                 precision: Precision = Precision.f64):
        self.config = c = config or CohereMelSpectrogram.Config()
        if c.cmvn_epsilon != 1.0e-5:
            raise ValueError("the CMVN epsilon of the device epilogue is CohereMelSpectrogram.Config's 1e-5")
        self.n_fft = 1 << max(0, (c.win_length - 1).bit_length())   # nextPowerOfTwo(atLeast: winLength)
        cfg = ex_config("cohere", sample_rate=c.sample_rate, win_length=c.win_length, hop_length=c.hop_length,
                        n_mels=c.n_mels, n_fft=self.n_fft, f_min=c.f_min, f_max=c.f_max, preemph=c.preemph,
                        spectrum_power=c.mag_power, log_floor=c.log_zero_guard)
        self.mel = AudioMelSpectrogram.from_ex_config(cfg, precision)

    def valid_frame_count(self, n: int) -> int:
        return max(0, n) // self.config.hop_length

    def features(self, audio, fixed_frames: int = 3_500) -> tuple[np.ndarray, int]:
        """``compute`` followed by ``padOrTruncate(fixedFrames:)`` in one call: ([nMels x fixedFrames], featureLength).
        ``fixed_frames < 0`` skips the padOrTruncate (then this is ``compute``)."""
        audio = np.ascontiguousarray(audio, np.float32).reshape(-1)
        n = audio.size
        W = 1 + n // self.config.hop_length if fixed_frames < 0 else int(fixed_frames)
        out = np.zeros((self.config.n_mels, W), np.float32)
        frames, valid = C.c_int64(), C.c_int64()
        _lib.check(self.mel._L.fa_mel_cohere_features(self.mel._h, _lib.ptr(audio) if n else None, n, int(fixed_frames),
                                                      out.ctypes.data, out.size, C.byref(frames), C.byref(valid)),
                   "fa_mel_cohere_features")
        return out, int(valid.value)

    def compute(self, audio) -> "CohereMelSpectrogram.Output":
        mel, valid = self.features(audio, -1)
        return CohereMelSpectrogram.Output(mel, valid)

    @staticmethod
    def pad_or_truncate(mel: np.ndarray, valid_frames: int, fixed_frames: int = 3_500) -> tuple[np.ndarray, int]:
        """``padOrTruncate`` (:250-263) on a [nMels x T] array."""
        mel = np.asarray(mel, np.float32)
        if mel.shape[0] == 0:
            return mel, 0
        cur = mel.shape[1]
        if cur >= fixed_frames:
            return mel[:, :fixed_frames].copy(), min(valid_frames, fixed_frames)
        pad = np.zeros((mel.shape[0], fixed_frames - cur), np.float32)
        return np.concatenate([mel, pad], axis=1), min(valid_frames, fixed_frames)


class StyleTTS2MelExtractor:
    """TTS/StyleTTS2/Pipeline/Preprocess/StyleTTS2MelExtractor.swift: torchaudio MelSpectrogram(n_mels 80, n_fft 2048,
    win 1200, hop 300) on 24 kHz audio with the HTK table built for 16 kHz bins, reflect padding, and
    ``(log(mel + 1e-5) - (-4)) / 4`` (``fa_mel_styletts2_features``: one kernel launch)."""

    def __init__(self, n_fft: int = 2048, win_length: int = 1200, hop_length: int = 300, n_mels: int = 80,
                 filter_sample_rate: int = 16_000, mean: float = -4.0, std: float = 4.0, log_epsilon: float = 1e-5,
                 sample_rate: int = 24_000):
        self.n_mels, self.hop_length = n_mels, hop_length
        cfg = ex_config("styletts2", n_fft=n_fft, win_length=win_length, hop_length=hop_length, n_mels=n_mels,
                        filter_sample_rate=filter_sample_rate, log_mean=mean, log_std=std, log_floor=log_epsilon,
                        sample_rate=sample_rate)
        self.mel = AudioMelSpectrogram.from_ex_config(cfg)

    def compute(self, audio) -> tuple[np.ndarray, int]:
        """(mel [nMels x frames] row-major, frames), frames = 1 + n / hop."""
        audio = np.ascontiguousarray(audio, np.float32).reshape(-1)
        n = audio.size
        T = 1 + n // self.hop_length
        out = np.empty((self.n_mels, T), np.float32)
        frames = C.c_int64()
        _lib.check(self.mel._L.fa_mel_styletts2_features(self.mel._h, _lib.ptr(audio) if n else None, n, out.ctypes.data,
                                                         out.size, C.byref(frames)), "fa_mel_styletts2_features")
        return out, int(frames.value)


class LuxTtsMelExtractor:
    """TTS/LuxTts/LuxTtsMelExtractor.swift: torchaudio MelSpectrogram(24000, n_fft 1024, hop 256, 100 mels, power 1,
    reflect padding) with the float64 HTK table, ``log(max(mel, 1e-7))`` and lhotse's frame count
    (``fa_mel_luxtts_features``: one kernel launch)."""

    def __init__(self):
        self.n_mels, self.hop_length = 100, 256
        self.mel = AudioMelSpectrogram.from_ex_config(ex_config("luxtts"))

    def frame_count(self, sample_count: int) -> int:
        """lhotse ``compute_num_frames``: (n + hop/2) / hop."""
        return (sample_count + self.hop_length // 2) // self.hop_length

    def extract(self, audio) -> np.ndarray:
        """[T x nMels] log-mel frames, T = frame_count(n) (none for an empty clip)."""
        audio = np.ascontiguousarray(audio, np.float32).reshape(-1)
        n = audio.size
        T = self.frame_count(n) if n else 0
        out = np.empty((T, self.n_mels), np.float32)
        frames = C.c_int64()
        _lib.check(self.mel._L.fa_mel_luxtts_features(self.mel._h, _lib.ptr(audio) if n else None, n,
                                                      out.ctypes.data if T else None, out.size, C.byref(frames)),
                   "fa_mel_luxtts_features")
        return out
