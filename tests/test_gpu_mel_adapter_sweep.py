"""The log-mel adapters against the oracle across their configuration space (GPU tests run with ``-m gpu`` on an H100).

``mel_adapters.cu`` holds three kernels behind three C entry points: ``per_feature_norm_kernel`` (UnifiedMelExtractor's
per-feature normalisation, transposed to [nMels x T] through a 128-bin x 32-frame shared tile, ``fa_mel_unified_features``),
``per_feature_norm_inplace_kernel`` (``fa_mel_normalize_per_feature``) and ``lseend_scale_cmn_kernel`` (LS-EEND's log10
scaling and running cumulative mean, ``fa_mel_lseend_features``).  They restate the reference's loops with individually
rounded float32 operations, so they are held to the oracle bit for bit:

* CPU: a numpy float32 restatement (frames in order, bins vectorised, every operation rounded to float32) equals
  ``oracle.normalize_per_feature`` and ``oracle.lseend_scale_cmn`` bit for bit.
* GPU, by composition on one handle, so that no mel error enters: ``fa_mel_unified_features(window, valid_count)`` equals
  ``oracle.normalize_per_feature(M_c, valid).T`` and the transpose of ``fa_mel_normalize_per_feature(M_c, valid)``, where
  ``M_c`` is the same handle's ``.center`` log-mel with expected count T = n / hop + 1; ``fa_mel_lseend_features`` equals
  ``oracle.lseend_scale_cmn(M_p, mean, count)`` (features, mean and count), ``M_p`` the handle's ``.prePadded`` log-mel.
  Equal means the same NaN positions and the same bits everywhere else.

End to end against the oracle's own log-mel the adapters inherit the mel error ``e`` (test_gpu_mel_sweep.py's bars:
1e-5 + 4e-7 |r| for the FP64 transform and the generic kernel, the float32-pair bar otherwise).  To first order:

* unified, element (t, m) of a column with spread sd (its unbiased std + 1e-5): |dz| <= (e_t + E)/sd + |z| sqrt(2) E/sd,
  E = max over the valid frames of e (the mean moves by at most E, the std by at most sqrt(n/(n-1)) E).  The bar is 1.25
  times that (second order: E/sd <= 0.05 where it is applied) plus each side's own float32 rounding, measured against a
  float64 evaluation of the same formula on that side's log-mel.  Columns with E > 0.05 sd make the bar meaningless; they
  are left to the bit-exact checks and counted, and the count must be 0 on the noise and speech fixtures (empty filters,
  whose columns are the constant log floor, are excluded as such).
* LS-EEND, frame t of a chain: |dy_t| <= s (e_t + max_{k<=t} e_k), s = 1 / ln 10 (the running mean is a weighted average
  of the scaled frames), plus each side's float32 rounding of the chain, measured the same way.
* Non-finite input: the library makes a NaN frame NaN in every non-empty band only, the oracle in every mel (DESIGN §2);
  overflowing power is non-finite in the library only where the oracle is.

The worst deviation seen, as a fraction of its bar, is printed per bar (run with ``-s``).  The ``.center`` mode with an
expected frame count, the mode UnifiedMelExtractor calls, is also checked on the plain mel entry points here.
"""
import ctypes as C
import math
import threading

import numpy as np
import pytest

from fluidaudio_b200 import _lib, synth
from fluidaudio_b200.mel import AudioMelSpectrogram, LogFloorMode, Precision

F32 = np.float32
CENTER, PRE_PADDED = 0, 1
TIME_MAJOR, MEL_MAJOR = 0, 1
INVALID_ARGUMENT = 1
SCALE = F32(1.0) / F32(math.log(10.0))         # LSEENDPreprocessor.swift:36, 1 / logf(10) in float32

UNIFIED_MELS = (1, 23, 80, 127, 128, 129, 255, 256, 257, 512)
UNIFIED_T = (1, 2, 31, 32, 33, 63, 64, 65, 300)
UNIFIED_HANDLES = {
    "default": dict(n_fft=512, win_length=400, hop_length=160),
    "nfft256": dict(n_fft=256, win_length=200, hop_length=80),
    "hop161": dict(n_fft=512, win_length=400, hop_length=161),
    "nfft1024": dict(n_fft=1024, win_length=1024, hop_length=256),
}
INPUTS = ("noise", "speech", "silence", "nan", "overflow")
WORST = {}                                      # largest |d| / bar per bar, printed at the end of each test


def _note(key, frac):
    WORST[key] = max(WORST.get(key, 0.0), float(frac))


def _report(title):
    print(f"\n{title}: worst |d| / bar " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


# ================================================================================================ float32 restatements
def np_normalize_per_feature(x, valid):
    """UnifiedMelExtractor.normalizePerFeature (UnifiedMelExtractor.swift:88-113) in numpy float32: frames in order,
    bins at once, every operation rounded to float32.  x: [frames x nMels]; 0 < valid <= frames, else all zero."""
    x = np.asarray(x, F32)
    out = np.zeros_like(x)
    if valid <= 0:
        return out
    with np.errstate(all="ignore"):
        mean = np.zeros(x.shape[1], F32)
        for t in range(valid):
            mean = mean + x[t]
        mean = mean / F32(valid)
        var_sum = np.zeros(x.shape[1], F32)
        for t in range(valid):
            d = x[t] - mean
            var_sum = var_sum + d * d
        sd = np.sqrt(var_sum / F32(valid - 1 if valid > 1 else 1)) + F32(1e-5)
        for t in range(valid):
            out[t] = (x[t] - mean) / sd
    return out


def np_lseend_scale_cmn(x, mean, count):
    """LSEENDPreprocessor.processAudioQueue's scaling and cumulative mean (:259-279) in numpy float32: per frame
    count += 1, alpha = 1 / Float(count), v = x * scale, mean = mean + alpha * (v - mean), x = v - mean."""
    x = np.asarray(x, F32)
    out = np.empty_like(x)
    mean = np.asarray(mean, F32).copy()
    with np.errstate(all="ignore"):
        for t in range(x.shape[0]):
            count += 1
            alpha = F32(1.0) / F32(count)
            v = x[t] * SCALE
            mean = mean + alpha * (v - mean)
            out[t] = v - mean
    return out, mean, count


def same_bits(a, b):
    """Same shape, NaN in the same places, the same bits everywhere else."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32)))


def _matrix(kind, T, M, seed):
    """[T x M] log-mel-like float32 values of one kind: noise, every column constant, columns whose variance sum (or
    sum) overflows float32, NaN / +-Inf entries."""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((T, M)) * 3 - 7).astype(F32)
    if kind == "constant" and T:
        x[:] = x[0]
    elif kind == "overflow":
        x[:, ::2] = (np.sign(x[:, ::2]) * F32(3e19)).astype(F32)      # (d * d) ~ 1e39: the variance sum overflows
        x[:, 1::4] = F32(2e38)                                         # the sum itself overflows from the second frame
    elif kind == "nonfinite" and T:
        x[rng.integers(0, T), ::3] = np.nan
        x[rng.integers(0, T), 1::3] = np.inf
        x[rng.integers(0, T), 2::5] = -np.inf
    return x


NORM_FRAMES = (0, 1, 31, 32, 33)
NORM_MELS = (1, 127, 128, 129, 1000)
MATRIX_KINDS = ("noise", "constant", "overflow", "nonfinite")


def _valids(T):
    return sorted({-3, 0, 1, 2, max(T - 1, 1), T, T + 5})


def test_float32_restatement_pins_the_oracle_adapters(oracle):
    """The oracle's C adapters equal an independent numpy float32 restatement bit for bit, on the shapes, valid counts,
    running counts and non-finite values the GPU sweep uses."""
    for T in NORM_FRAMES:
        for M in NORM_MELS:
            for kind in MATRIX_KINDS:
                x = _matrix(kind, T, M, seed=T * 1000 + M)
                for valid in _valids(T):
                    v = min(valid, T)
                    assert same_bits(oracle.normalize_per_feature(x, v), np_normalize_per_feature(x, v)), (T, M, kind, v)
    for M in (1, 23, 80, 128, 129):
        for count in (0, 2 ** 24 - 3, 2 ** 31 + 5):
            for kind, mean_kind in (("noise", "zero"), ("noise", "noise"), ("nonfinite", "noise"), ("noise", "nan"),
                                    ("noise", "inf")):
                for T in (0, 1, 7, 33):
                    x = _matrix(kind, T, M, seed=M + T)
                    mean = _mean_in(mean_kind, M, seed=T)
                    got = oracle.lseend_scale_cmn(x, mean, count)
                    want = np_lseend_scale_cmn(x, mean, count)
                    what = (M, count, kind, mean_kind, T)
                    assert same_bits(got[0], want[0]) and same_bits(got[1], want[1]) and got[2] == want[2] == count + T, what
    # the chained oracle entry point is the scaling applied to the oracle's own .prePadded log-mel
    cfg = oracle.lseend_config()
    a = synth.tone_noise_audio(9000)
    mel, ml, _ = oracle.mel_flat_transposed(cfg, a, 0.0, 1, None)
    f, mean, cnt = oracle.lseend_features(cfg, a, np.zeros(23, F32), 5)
    g = np_lseend_scale_cmn(mel[:ml], np.zeros(23, F32), 5)
    assert same_bits(f, g[0]) and same_bits(mean, g[1]) and cnt == g[2]


def _mean_in(kind, M, seed):
    rng = np.random.default_rng(seed + 77)
    mean = np.zeros(M, F32) if kind == "zero" else (rng.standard_normal(M) * 2 - 3).astype(F32)
    if kind == "nan":
        mean[::2] = np.nan
    elif kind == "inf":
        mean[::2] = np.inf
        mean[1::4] = -np.inf
    return mean


def test_oracle_unified_features_take_a_full_config(oracle):
    """``cfg=`` restates any handle's configuration; the default call is unchanged, and an empty window gives the reference
    guard's single zero frame."""
    a = synth.tone_noise_audio(8000)
    m0, v0 = oracle.unified_mel_features(a, 6000)
    m1, v1 = oracle.unified_mel_features(a, 6000, cfg=oracle.mel_config(n_mels=128))
    assert v0 == v1 and m0.tobytes() == m1.tobytes()
    cfg = oracle.mel_config(n_mels=40, n_fft=256, win_length=200, hop_length=80)
    m2, v2 = oracle.unified_mel_features(a, 6000, cfg=cfg)
    raw, _, _ = oracle.mel_flat_transposed(cfg, a, 0.0, 0, expected_frames=8000 // 80 + 1)
    assert v2 == 75 and m2.shape == (40, 101)
    assert same_bits(m2, np_normalize_per_feature(raw, 75).T)
    m3, v3 = oracle.unified_mel_features(np.zeros(0, F32), 500, cfg=cfg)
    assert v3 == 1 and m3.shape == (40, 1) and not m3.any()


# ================================================================================================ GPU helpers
def _kind_of(m):
    """mel_generic_kernel ignores the precision switch, the specialised kernel's two transforms never agree on noise."""
    probe = synth.tone_noise_audio(16000, seed=1)
    prec, outs = m.precision, []
    for p in (Precision.f64, Precision.f32):
        m.set_precision(p)
        outs.append(m.compute_flat_transposed(probe)[0].copy())
    m.set_precision(prec)
    return "generic" if np.array_equal(outs[0], outs[1]) else "mel512"


def fp64_bar(r, top):                       # test_gpu_mel_sweep.py's bars (DESIGN §4.1)
    return 1e-5 + 4e-7 * np.abs(r)


def f32_bar(r, top):
    return np.minimum(2e-3, 1e-4 * np.maximum(1.0, np.exp(top - r - 12.0)))


def _bar_for(kind, precision):
    return f32_bar if kind == "mel512" and precision == Precision.f32 else fp64_bar


def _bar_name(kind, precision):
    return "f32" if kind == "mel512" and precision == Precision.f32 else "fp64"


def _mel_bar(bar, mel):
    """Per-element mel bar of an oracle log-mel [T x M]; non-finite entries get an infinite bar."""
    fin = np.isfinite(mel)
    top = np.where(fin, mel, -np.inf).max(axis=1, keepdims=True) if mel.size else np.zeros((mel.shape[0], 1))
    with np.errstate(all="ignore"):
        e = bar(np.where(fin, mel, 0.0).astype(np.float64), np.broadcast_to(top, mel.shape).astype(np.float64))
    return np.where(fin, e, np.inf)


def _audio(kind, n, seed):
    if kind == "speech":
        return synth.speech_like_audio(n, seed=seed)
    if kind == "silence":
        return np.zeros(n, F32)
    x = synth.tone_noise_audio(n, seed=seed)
    if kind == "nan" and n:
        x[n // 3] = np.nan
    elif kind == "overflow" and n:
        x[n // 4:n // 4 + max(1, n // 8)] *= F32(1e25)
        x[(3 * n) // 4] = np.inf
    return x


def unified(m, window, valid_count):
    """fa_mel_unified_features on handle m: ([nMels x T], valid); no float past T * nMels is written."""
    T = window.size // m.hop_length + 1
    out = np.full(T * m.n_mels + 8, 7.0, F32)
    tot, val = C.c_int64(), C.c_int32()
    _lib.check(m._L.fa_mel_unified_features(m._h, window.ctypes.data if window.size else None, window.size, int(valid_count),
                                            out.ctypes.data, T * m.n_mels, C.byref(tot), C.byref(val)),
               "fa_mel_unified_features")
    assert tot.value == T and (out[T * m.n_mels:] == 7.0).all()
    return out[:T * m.n_mels].reshape(m.n_mels, T), val.value


def center_mel(m, window, T):
    """The handle's own .center log-mel with expected frame count T, time-major [T x nMels]."""
    out, ml, nf = m._run(window, 0.0, CENTER, T, TIME_MAJOR)
    assert nf == T
    return out[:T * m.n_mels].reshape(T, m.n_mels)


def lseend(m, chunk, mean, count):
    """fa_mel_lseend_features on handle m: (features [T x nMels], mean', count')."""
    T = m.frame_count(chunk.size, PRE_PADDED)
    out = np.full(max(T, 0) * m.n_mels + 8, 7.0, F32)
    mean = np.ascontiguousarray(mean, F32).copy()
    cnt, frames = C.c_int64(count), C.c_int64()
    _lib.check(m._L.fa_mel_lseend_features(m._h, chunk.ctypes.data if chunk.size else None, chunk.size, mean.ctypes.data,
                                           C.byref(cnt), out.ctypes.data, max(T, 0) * m.n_mels, C.byref(frames)),
               "fa_mel_lseend_features")
    assert frames.value == max(T, 0) and (out[frames.value * m.n_mels:] == 7.0).all()
    return out[:frames.value * m.n_mels].reshape(frames.value, m.n_mels), mean, cnt.value


def prepadded_mel(m, chunk):
    T = max(m.frame_count(chunk.size, PRE_PADDED), 0)
    if T == 0:
        return np.zeros((0, m.n_mels), F32)
    out, ml, nf = m._run(chunk, 0.0, PRE_PADDED, None, TIME_MAJOR)
    assert ml == nf == T
    return out[:T * m.n_mels].reshape(T, m.n_mels)


def standalone_norm(x, valid):
    y = np.ascontiguousarray(x, F32).copy()
    _lib.check(_lib.load().fa_mel_normalize_per_feature(y.ctypes.data, y.shape[0], y.shape[1], int(valid)),
               "fa_mel_normalize_per_feature")
    return y


def lseend_handle(sample_rate=16000, n_mels=23, win_length=400, hop_length=160):
    """LSEENDPreprocessor's AudioMelSpectrogram (:70-81) for model metadata: nFFT = nextPow2(winLength)
    (LSEENDTypes.swift:55-57)."""
    n_fft = 1 << (win_length - 1).bit_length()
    kw = dict(sample_rate=sample_rate, n_mels=n_mels, n_fft=n_fft, hop_length=hop_length, win_length=win_length,
              preemph=0.0, pad_to=0, log_floor=1e-10, log_floor_mode=LogFloorMode.clamped, window_periodic=True)
    return AudioMelSpectrogram(**kw), kw


# ================================================================================================ D: end-to-end bars
def _norm64(mel, valid):
    """The normalisation in float64 on the same log-mel: [valid x M] z and the column's sd."""
    x = mel[:valid].astype(np.float64)
    with np.errstate(all="ignore"):
        sd = np.sqrt(((x - x.mean(axis=0)) ** 2).sum(axis=0) / max(valid - 1, 1)) + 1e-5
        return (x - x.mean(axis=0)) / sd, sd


def check_unified_end_to_end(got, lib_mel, ref, ref_mel, valid, band, bar, key, what, nan_input=False):
    """got / ref: [M x T] features of the library and the oracle; lib_mel / ref_mel: the [T x M] log-mel each normalised.
    nan_input: the window holds a NaN sample (and no overflow).  Returns the number of non-empty-band columns left out
    for a tiny spread."""
    assert not (~np.isfinite(got) & np.isfinite(ref)).any(), (what, "non-finite where the oracle is finite")
    if nan_input:
        assert np.array_equal(np.isnan(got), np.isnan(ref) & band[:, None]), (what, "NaN footprint")
    assert not got[:, max(valid, 0):].any() and not ref[:, max(valid, 0):].any(), what
    if valid <= 1:
        fin = np.isfinite(got) & np.isfinite(ref)
        assert np.array_equal(got[fin], ref[fin]), what
        return 0
    cols = band & np.isfinite(ref_mel[:valid]).all(axis=0) & np.isfinite(lib_mel[:valid]).all(axis=0)
    e = _mel_bar(bar, ref_mel[:valid])
    E = e.max(axis=0)
    z_ref, sd = _norm64(ref_mel, valid)
    z_lib, _ = _norm64(lib_mel, valid)
    tiny = cols & (E > 0.05 * sd)
    use = cols & ~tiny
    if use.any():
        g, r = got[use, :valid].T.astype(np.float64), ref[use, :valid].T.astype(np.float64)
        first = (e[:, use] + E[use]) / sd[use] + np.abs(z_ref[:, use]) * math.sqrt(2.0) * E[use] / sd[use]
        limit = 1.25 * first + np.abs(g - z_lib[:, use]) + np.abs(r - z_ref[:, use]) + 1e-12
        d = np.abs(g - r)
        frac = (d / limit).max()
        _note(key, frac)
        assert frac <= 1.0, (what, "worst |d| / bar", float(frac), "max |d|", float(d.max()))
    return int(tiny.sum())


def _cmn64(mel, mean0, count0):
    """LS-EEND scaling and cumulative mean in float64 on the same log-mel."""
    y = mel.astype(np.float64) * float(SCALE)
    out, mean = np.empty_like(y), mean0.astype(np.float64)
    for t in range(y.shape[0]):
        mean = mean + (y[t] - mean) / (count0 + t + 1)
        out[t] = y[t] - mean
    return out


def check_lseend_end_to_end(got, lib_mel, ref, ref_mel, bar, key, what):
    """Whole chains from a zero state: got / ref features [N x M], lib_mel / ref_mel the log-mel each side scaled."""
    assert got.shape == ref.shape and np.isfinite(ref).all() and np.isfinite(got).all(), what
    if not got.size:
        return
    e = _mel_bar(bar, ref_mel)
    first = float(SCALE) * (e + np.maximum.accumulate(e, axis=0))
    zero = np.zeros(got.shape[1])
    limit = first + np.abs(got - _cmn64(lib_mel, zero, 0)) + np.abs(ref - _cmn64(ref_mel, zero, 0)) + 1e-12
    frac = (np.abs(got.astype(np.float64) - ref) / limit).max()
    _note(key, frac)
    assert frac <= 1.0, (what, "worst |d| / bar", float(frac))


# ================================================================================================ B/C/D: unified
@pytest.mark.gpu
@pytest.mark.parametrize("handle", list(UNIFIED_HANDLES))
def test_unified_features_bitwise_and_end_to_end(gpu_lib, oracle, handle):
    """fa_mel_unified_features over n_mels on both sides of every 128-bin CTA edge, T on both sides of the 32-frame tile
    edges, window_samples = (T - 1) hop + r (r = 0, hop - 1; T = 1, r = 0 is the empty window), valid 0 / 1 / 2 / T - 1 / T
    / clamped, both precisions and every input kind: bit for bit against the oracle's normalisation of the handle's own
    log-mel and against the standalone kernel, then end to end against the oracle within the derived bar."""
    hk = UNIFIED_HANDLES[handle]
    hop = hk["hop_length"]
    tiny_counts = {}
    for i, nm in enumerate(UNIFIED_MELS):
        kw = dict(sample_rate=16000, n_mels=nm, preemph=0.97, pad_to=0, window_periodic=False, **hk)
        m = AudioMelSpectrogram(**kw)
        kind = _kind_of(m)
        if handle == "default":
            assert kind == "mel512"
        else:
            assert kind == "generic", handle
        cfg = oracle.mel_config(**kw)
        band = oracle.mel_filterbank(hk["n_fft"], nm, 16000).any(axis=1)
        for j, T in enumerate(UNIFIED_T):
            for r in (0, hop - 1):
                n = (T - 1) * hop + r
                src = INPUTS[(i + 2 * j + (r > 0)) % len(INPUTS)]
                window = _audio(src, n, seed=i * 31 + T + r)
                valid_counts = (hop - 1, hop, 2 * hop + 1, n, T * hop, n + 10 * hop)
                ref_mel = oracle.mel_flat_transposed(cfg, window, 0.0, 0, expected_frames=T)[0].reshape(-1, nm)
                assert ref_mel.shape == (T, nm)
                for prec in (Precision.f64, Precision.f32):
                    m.set_precision(prec)
                    bar, key = _bar_for(kind, prec), f"unified {_bar_name(kind, prec)}"
                    M_c = center_mel(m, window, T)
                    for k, vc in enumerate(valid_counts):
                        what = dict(handle=handle, n_mels=nm, T=T, n=n, valid_count=vc, input=src, precision=int(prec))
                        valid = min(vc // hop, T)
                        got, v = unified(m, window, vc)
                        assert v == valid, what
                        # B: bit for bit by composition
                        assert same_bits(got, oracle.normalize_per_feature(M_c, valid).T), what
                        assert same_bits(got, standalone_norm(M_c, valid).T), what
                        # D: end to end against the oracle's own log-mel
                        ref = oracle.normalize_per_feature(ref_mel, valid).T
                        if k == 0 and prec == Precision.f64 and T < 100:
                            rm, rv = oracle.unified_mel_features(window, vc, cfg=cfg)
                            assert rv == valid and same_bits(rm, ref), what
                        tiny = check_unified_end_to_end(got, M_c, ref, ref_mel, valid, band, bar, key, what,
                                                        nan_input=src == "nan")
                        if src in ("noise", "speech") and valid >= 16:
                            tiny_counts[(nm, T, r, int(prec), vc)] = tiny
        m.close()
    assert tiny_counts and not any(tiny_counts.values()), {k: v for k, v in tiny_counts.items() if v}
    _report(f"unified {handle}")


# ================================================================================================ B/C: standalone
@pytest.mark.gpu
def test_standalone_normalisation_bitwise(gpu_lib, oracle):
    """fa_mel_normalize_per_feature at frames 0 / 1 / 31 / 32 / 33 x n_mels 1 / 127 / 128 / 129 / 1000, valid <= 0 (a host
    memset, no launch), inside and past the frame count (clamped), on noise, constant columns, overflowing variance sums
    and NaN / Inf entries: bit for bit against the oracle."""
    for T in NORM_FRAMES:
        for M in NORM_MELS:
            for kind in MATRIX_KINDS:
                x = _matrix(kind, T, M, seed=T * 1000 + M)
                for valid in _valids(T):
                    before = _lib.kernel_launch_count()
                    got = standalone_norm(x, valid)
                    launches = _lib.kernel_launch_count() - before
                    assert launches == (1 if T > 0 and valid > 0 else 0), (T, M, valid, launches)
                    want = oracle.normalize_per_feature(x, min(valid, T)) if valid > 0 else np.zeros_like(x)
                    assert same_bits(got, want), (T, M, kind, valid)


# ================================================================================================ B/C/D: LS-EEND
class ChunkQueue:
    """StreamingChunkQueue (LSEENDPreprocessor.swift:290-376) for audio (stride 1): leftContext zeros seeded, popAllChunks
    returns every whole chunk at once with its context."""

    def __init__(self, chunk, left, right):
        self.chunk, self.context = chunk, left + right
        self.buffer = np.zeros(left, F32)
        self.head = 0

    def append(self, x):
        self.buffer = np.concatenate([self.buffer, np.asarray(x, F32)])

    def unread(self):
        return self.buffer.size - self.head

    def pop_all(self):
        if self.unread() < self.chunk + self.context:
            return None
        new_head = self.head + (self.buffer.size - self.head - self.context) // self.chunk * self.chunk
        out = self.buffer[self.head:new_head + self.context].copy()
        self.head = new_head
        return out


def lseend_chunks(audio, n_fft, hop, seed, subsampling=10, chunk_size=2, context=7, conv_delay=2):
    """The chunks LSEENDPreprocessor pops (:56-60, :100-105, :158-180, :249-251) when `audio` arrives in random sizes and
    ends with drainRightContextWithSilence: k * chunkSamples + nFFT - hop samples each."""
    chunk_samples = hop * subsampling * chunk_size
    q = ChunkQueue(chunk_samples, n_fft // 2, n_fft // 2 - hop)
    rng = np.random.default_rng(seed)
    out, pos = [], 0
    while pos < audio.size:
        step = int(rng.integers(0, 3 * chunk_samples))
        q.append(audio[pos:pos + step])
        pos += step
        c = q.pop_all()
        if c is not None:
            out.append(c)
    q.append(np.zeros((context + conv_delay * subsampling) * hop + n_fft // 2, F32))
    over = max(0, q.unread() - q.context)
    q.append(np.zeros((chunk_samples - over % chunk_samples) % chunk_samples, F32))
    c = q.pop_all()
    if c is not None:
        out.append(c)
    for c in out:
        assert (c.size - (n_fft - hop)) % chunk_samples == 0 and c.size > n_fft - hop
    return out


LSEEND_CONFIGS = {
    "16k": dict(sample_rate=16000, n_mels=23, win_length=400, hop_length=160),
    "8k": dict(sample_rate=8000, n_mels=23, win_length=200, hop_length=80),
    "mels80": dict(sample_rate=16000, n_mels=80, win_length=400, hop_length=160),
    "mels128": dict(sample_rate=16000, n_mels=128, win_length=400, hop_length=160),
    "mels129": dict(sample_rate=16000, n_mels=129, win_length=400, hop_length=160),
    "odd_hop": dict(sample_rate=16000, n_mels=40, win_length=400, hop_length=161),
}


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(LSEEND_CONFIGS))
def test_lseend_features_bitwise_and_end_to_end(gpu_lib, oracle, config):
    """fa_mel_lseend_features on the preprocessor's chunk sequences (random arrival sizes, drained with silence), both
    precisions: features, mean and count bit for bit against the oracle's scaling of the handle's own .prePadded log-mel;
    the whole chain against a chain of oracle.lseend_features within the derived bar.  Direct edges: 0 samples, fewer
    than nFFT - hop (no frame, no launch, state untouched), nFFT - 1 (one frame), running counts 0 / 2^24 - 3 / 2^31 + 5,
    NaN and Inf already in the running mean."""
    m, kw = lseend_handle(**LSEEND_CONFIGS[config])
    n_fft, hop, nm = kw["n_fft"], kw["hop_length"], kw["n_mels"]
    kind = _kind_of(m)
    assert kind == ("mel512" if n_fft == 512 and hop % 2 == 0 else "generic"), config
    cfg = oracle.lseend_config(n_mels=nm, n_fft=n_fft, hop_length=hop, win_length=kw["win_length"],
                               sample_rate=kw["sample_rate"])
    sr = kw["sample_rate"]
    for src, seed in (("noise", 1), ("speech", 2)):
        audio = _audio(src, 3 * sr + 123, seed=seed)
        chunks = lseend_chunks(audio, n_fft, hop, seed=seed)
        assert len(chunks) >= 3
        ref_f, ref_m, mean_r, cnt_r = [], [], np.zeros(nm, F32), 0
        for c in chunks:
            f, mean_r, cnt_r = oracle.lseend_features(cfg, c, mean_r, cnt_r)
            ref_f.append(f)
            ref_m.append(oracle.mel_flat_transposed(cfg, c, 0.0, 1, None)[0].reshape(-1, nm))
        for prec in (Precision.f64, Precision.f32):
            m.set_precision(prec)
            mean, cnt, feats, mels = np.zeros(nm, F32), 0, [], []
            for i, c in enumerate(chunks):
                M_p = prepadded_mel(m, c)
                want = oracle.lseend_scale_cmn(M_p, mean, cnt)
                f, mean, cnt = lseend(m, c, mean, cnt)
                what = dict(config=config, input=src, chunk=i, n=c.size, precision=int(prec))
                assert same_bits(f, want[0]) and same_bits(mean, want[1]) and cnt == want[2], what
                feats.append(f)
                mels.append(M_p)
            assert cnt == cnt_r
            check_lseend_end_to_end(np.concatenate(feats), np.concatenate(mels), np.concatenate(ref_f),
                                    np.concatenate(ref_m), _bar_for(kind, prec), f"lseend {_bar_name(kind, prec)}",
                                    dict(config=config, input=src, precision=int(prec)))
    # direct edges
    a = synth.tone_noise_audio(40 * hop + n_fft, seed=5)
    for prec in (Precision.f64, Precision.f32):
        m.set_precision(prec)
        for n in (0, 1, n_fft - hop - 1, n_fft - hop):
            mean = _mean_in("noise", nm, seed=n)
            before = _lib.kernel_launch_count()
            f, mean2, cnt = lseend(m, a[:n], mean, 1234)
            assert _lib.kernel_launch_count() == before and f.shape == (0, nm), (config, n)
            assert mean2.tobytes() == mean.tobytes() and cnt == 1234
        f, _, cnt = lseend(m, a[:n_fft - 1], np.zeros(nm, F32), 0)
        assert f.shape == (1, nm) and cnt == 1                         # (n - nFFT) / hop truncates toward zero
        for count in (0, 2 ** 24 - 3, 2 ** 31 + 5):
            for mean_kind in ("zero", "noise", "nan", "inf"):
                for n in (n_fft - 1, n_fft - hop + 1, 7 * hop + n_fft, 40 * hop + n_fft):
                    c = a[:n]
                    mean = _mean_in(mean_kind, nm, seed=n)
                    want = oracle.lseend_scale_cmn(prepadded_mel(m, c), mean, count)
                    f, mean2, cnt = lseend(m, c, mean, count)
                    what = dict(config=config, count=count, mean=mean_kind, n=n, precision=int(prec))
                    assert same_bits(f, want[0]) and same_bits(mean2, want[1]) and cnt == want[2], what
    m.close()
    _report(f"lseend {config}")


# ================================================================================================ E: .center + expected
def compare_mel(got, ref, fb, bar, key, what):
    """test_gpu_mel_sweep.py's comparison: oracle NaN frames are NaN in every non-empty band, non-finite values equal,
    the rest within the bar."""
    nan_rows = np.isnan(ref).any(axis=1)
    band = fb.any(axis=1)
    assert np.isnan(got[nan_rows][:, band]).all(), what
    g, r = got[~nan_rows], ref[~nan_rows]
    fin = np.isfinite(r)
    assert np.array_equal(g[~fin], r[~fin]) and np.isfinite(g[fin]).all(), what
    if fin.any():
        top = np.broadcast_to(np.where(fin, r, -np.inf).max(axis=1, keepdims=True), r.shape)
        frac = (np.abs(g[fin] - r[fin]) / bar(r[fin], top[fin])).max()
        _note(key, frac)
        assert frac <= 1.0, (what, float(frac))


@pytest.mark.gpu
def test_center_with_expected_frames_on_the_mel_entry_points(gpu_lib, oracle):
    """The mode UnifiedMelExtractor calls: .center with an expected frame count below, equal to and above the computed
    count (frames past the padded end are the log floor), through fa_mel_compute with one unit, with four pipeline units
    on a long clip, and through fa_mel_compute_device; mel-major is the transpose of time-major bit for bit."""
    for kw in (dict(n_mels=80), dict(n_mels=129, hop_length=161), dict(n_mels=40, n_fft=256, win_length=200, hop_length=80)):
        m = AudioMelSpectrogram(**kw)
        kind = _kind_of(m)
        nm = kw["n_mels"]
        cfg = oracle.mel_config(**kw)
        fb = oracle.mel_filterbank(kw.get("n_fft", 512), nm)
        hop = kw.get("hop_length", 160)
        for n, chunks in ((16000 + 37, 1), (16500 * hop + 77, 4)):
            if chunks == 4 and kw.get("n_fft") == 256:
                continue
            x = synth.tone_noise_audio(n, seed=n % 97)
            computed = m.frame_count(n, CENTER)
            _lib.check(m._L.fa_mel_set_pipeline_chunks(m._h, chunks), "fa_mel_set_pipeline_chunks")
            for expected in (computed - 3, computed, computed + 5):
                ref, rml, rnf = oracle.mel_flat_transposed(cfg, x, 0.25, CENTER, expected_frames=expected)
                ref = ref.reshape(rnf, nm)
                assert rml == rnf == expected
                if expected > computed:                  # the last frame lies wholly past the padded end: the log floor
                    assert np.unique(ref[-1]).size == 1 and abs(float(ref[-1, 0]) - math.log(2.0 ** -24)) < 1e-5
                for prec in (Precision.f64, Precision.f32):
                    m.set_precision(prec)
                    what = dict(kw, n=n, chunks=chunks, expected=expected, precision=int(prec))
                    key = f"mel .center expected {_bar_name(kind, prec)}"
                    tm, ml, nf = m._run(x, 0.25, CENTER, expected, TIME_MAJOR)
                    assert (ml, nf) == (rml, rnf), what
                    tm = tm[:nf * nm].reshape(nf, nm)
                    compare_mel(tm, ref, fb, _bar_for(kind, prec), key, what)
                    mm, ml2, nf2 = m._run(x, 0.25, CENTER, expected, MEL_MAJOR)
                    assert (ml2, nf2) == (ml, nf) and np.array_equal(mm[:nf * nm].reshape(nm, nf), tm.T), what
                    if chunks == 1:
                        d_in = _lib.DeviceBuffer(x.nbytes + 64)
                        d_in.upload(x)
                        d_out = _lib.DeviceBuffer(nf * nm * 4 + 64)
                        for time_major, host in ((True, tm), (False, tm.T)):
                            res = m.compute_device(d_in, n, d_out, last_audio_sample=0.25, padding_mode=CENTER,
                                                   expected_frame_count=expected, time_major=time_major)
                            _lib.synchronize()
                            assert res == (ml, nf), what
                            dev = d_out.download((nf * nm,), F32).reshape(host.shape)
                            assert np.array_equal(dev, host), (what, time_major)
                        d_in.free()
                        d_out.free()
        m.close()
    _report("mel .center with expected")


# ================================================================================================ F: state and reuse
@pytest.mark.gpu
def test_adapter_state_and_reuse(gpu_lib):
    """A small unified window after a large one on the same handle equals a fresh handle's result (the staging is reused);
    an LS-EEND chain interleaved with compute_flat_transposed and unified calls on its handle equals the chain alone; two
    handles on two threads give their sequential results."""
    big = synth.speech_like_audio(300 * 160, seed=3)
    small = synth.tone_noise_audio(31 * 160 + 7, seed=4)
    for prec in (Precision.f64, Precision.f32):
        m = AudioMelSpectrogram(n_mels=257, precision=prec)
        unified(m, big, big.size)
        reused = unified(m, small, small.size - 900)
        fresh_h = AudioMelSpectrogram(n_mels=257, precision=prec)
        fresh = unified(fresh_h, small, small.size - 900)
        assert reused[1] == fresh[1] and same_bits(reused[0], fresh[0]), prec
        m.close()
        fresh_h.close()

    audio = synth.speech_like_audio(3 * 16000, seed=8)
    chunks = lseend_chunks(audio, 512, 160, seed=8)

    def chain(m, interleave):
        mean, cnt, outs = np.zeros(m.n_mels, F32), 0, []
        for i, c in enumerate(chunks):
            if interleave:
                m.compute_flat_transposed(audio[: 4000 + 999 * i])
                unified(m, audio[: 20000 + 1600 * i], 9000 + 160 * i)
            f, mean, cnt = lseend(m, c, mean, cnt)
            outs.append(f)
        return np.concatenate(outs), mean, cnt

    for prec in (Precision.f64, Precision.f32):
        m, _ = lseend_handle()
        m.set_precision(prec)
        plain = chain(m, False)
        mixed = chain(m, True)
        assert same_bits(plain[0], mixed[0]) and same_bits(plain[1], mixed[1]) and plain[2] == mixed[2], prec
        m.close()

    def work(m, results, slot):
        res = []
        for k in range(6):
            res.append(unified(m, big[: 8000 + 5000 * k], 6000 + 4000 * k)[0])
            res.append(lseend(m, chunks[k % len(chunks)], np.zeros(m.n_mels, F32), k)[0])
        results[slot] = res

    handles = [AudioMelSpectrogram(n_mels=128), AudioMelSpectrogram(n_mels=80, hop_length=161, precision=Precision.f32)]
    sequential = [None, None]
    for i, h in enumerate(handles):
        work(h, sequential, i)
    threaded = [None, None]
    threads = [threading.Thread(target=work, args=(h, threaded, i)) for i, h in enumerate(handles)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for i in range(2):
        assert threaded[i] is not None and len(threaded[i]) == len(sequential[i])
        assert all(same_bits(a, b) for a, b in zip(threaded[i], sequential[i])), i
    for h in handles:
        h.close()


# ================================================================================================ pad_to contract
@pytest.mark.gpu
def test_adapters_refuse_a_padded_handle(gpu_lib):
    """Both adapters return exactly their frames, so a handle with pad_to > 1 is refused with FA_STATUS_INVALID_ARGUMENT
    naming pad_to, before any copy or launch, the caller's buffers and the LS-EEND state untouched; pad_to 0 and 1
    work.  Also when T happens to be a multiple of pad_to."""
    L = _lib.load()
    a = synth.tone_noise_audio(16000, seed=2)
    for pad_to in (0, 1, 3, 8):
        m = AudioMelSpectrogram(n_mels=80, pad_to=pad_to)
        for n in (4000, 4800, 5000):                  # T = 26, 31, 32: some multiples of 8, some not
            T = n // 160 + 1
            out = np.full(T * 80, 7.0, F32)
            tot, val = C.c_int64(-1), C.c_int32(-1)
            before = _lib.kernel_launch_count()
            st = L.fa_mel_unified_features(m._h, a.ctypes.data, n, n, out.ctypes.data, out.size, C.byref(tot), C.byref(val))
            if pad_to <= 1:
                assert st == 0 and tot.value == T and val.value == T - 1
                continue
            assert st == INVALID_ARGUMENT, (pad_to, n, st, L.fa_last_error())
            assert b"pad_to" in L.fa_last_error(), L.fa_last_error()
            assert _lib.kernel_launch_count() == before and (out == 7.0).all()
        lm = AudioMelSpectrogram(n_mels=23, preemph=0.0, pad_to=pad_to, log_floor=1e-10, log_floor_mode=LogFloorMode.clamped,
                                 window_periodic=True)
        for n in (8352, 5312):                         # T = 50, 31
            T = (n - 512) // 160 + 1
            out = np.full(T * 23, 7.0, F32)
            mean = _mean_in("noise", 23, seed=n)
            keep = mean.copy()
            cnt, frames = C.c_int64(41), C.c_int64(-1)
            before = _lib.kernel_launch_count()
            st = L.fa_mel_lseend_features(lm._h, a.ctypes.data, n, mean.ctypes.data, C.byref(cnt), out.ctypes.data,
                                          out.size, C.byref(frames))
            if pad_to <= 1:
                assert st == 0 and frames.value == T and cnt.value == 41 + T
                continue
            assert st == INVALID_ARGUMENT, (pad_to, n, st, L.fa_last_error())
            assert b"pad_to" in L.fa_last_error()
            assert _lib.kernel_launch_count() == before and (out == 7.0).all()
            assert cnt.value == 41 and mean.tobytes() == keep.tobytes()
        m.close()
        lm.close()
