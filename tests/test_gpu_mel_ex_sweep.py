"""The torch-style log-mel frontends across their configuration space on the H100 (``-m gpu``), against the float64
restatement and the derived per-entry bar of tests/mel_ex_restated.py.

a. Variant matrix: every (kReflect, kSpectrum, kAffine) variant of ``mel_generic_kernel`` at >= 3 handles dealt round
   robin over table kind, nFFT 32 .. 4096, window, hop, mels, p, log floor, (mean, std), rate and pad_to; clip lengths
   from 0 to ~2 s, six signals, all three modes, both layouts, a nonzero ``last``.  The test restates the routing rules
   (MelPlan::init, MelPlan::launch) to count the calls per variant, and checks the bar's ceiling at each frame's
   strongest mel.  That ceiling is below the old 1e-4 bar wherever the strongest band spans at most 16 bin quads;
   a wider band (1 to 3 mels at nFFT 4096) carries the fmaf chain's worst case (4 nq + 1)u and can exceed 1e-4.
b. Cohere's preset on ``mel512_kernel``: FP64 held to the bar, float32 with the bar's float32-transform term.
c. The class entry points at non-preset parameters: the library within the bar of the restatement and ``oracle_torch``
   within the same bar (so the two differ by at most twice the bar); Cohere's features against ``oracle_torch`` with
   the first-order CMVN bar of test_gpu_mel_torch_sweep.py, whose log-mel budget is twice the derived bar here: the
   generic-kernel bar it uses for the preset does not cover |X| (measured 1.5 of it at mag_power 1).
d. ``cohere_cmvn_kernel`` bit for bit against ``oracle_torch.cohere_cmvn`` of the handle's own log-mel, for mel counts
   that leave partial CTAs and warps.
e. Bitwise invariants for the 12 variants: layouts, batches, device buffers, pipeline units, and ``fa_audio_to_mel``
   against ``fa_mel_compute`` of ``fa_audio_resample`` on converted PCM that runs in several units.
f. Non-finite footprints for every variant.
"""
import ctypes as C
import time

import numpy as np
import pytest

import mel_ex_restated as R
from fluidaudio_b200 import _lib
from fluidaudio_b200.audio_converter import AudioConverter
from fluidaudio_b200.mel import (AudioMelSpectrogram, CohereMelSpectrogram, LuxTtsMelExtractor, Precision,
                                 StyleTTS2MelExtractor, ex_config)
from mel_ex_restated import CENTER, LEGACY, PRE_PADDED, Cfg
from oracle import oracle_torch as OT
from test_gpu_mel_torch_sweep import cmvn_frac, same_bits

pytestmark = pytest.mark.gpu
F32 = np.float32
TIME_MAJOR, MEL_MAJOR = 0, 1
WORST = {}
T0 = time.time()


def _note(key, frac):
    WORST[key] = max(WORST.get(key, 0.0), float(frac))


def handle(cfg: Cfg, precision=Precision.f64) -> AudioMelSpectrogram:
    return AudioMelSpectrogram.from_ex_config(ex_config(None, **cfg.ex_fields()), precision)


def run(mel, cfg, a, mode, last=0.0, layout=TIME_MAJOR, expected=None):
    """fa_mel_compute: ([Tp x M] time-major float32, T, Tp)."""
    out, ml, nf = mel._run(a, last, mode, expected, layout)
    x = out[:nf * cfg.n_mels]
    x = x.reshape(nf, cfg.n_mels) if layout == TIME_MAJOR else x.reshape(cfg.n_mels, nf).T
    return x, ml, nf


def restated(mel, cfg, a, mode, last=0.0, T=None):
    return R.restate(cfg, mel.get_hann_window(), mel.get_filterbank(), a, mode, last, T)


# ================================================================================================ a. variant matrix
def test_variant_matrix_against_the_restatement(gpu_lib):
    t0 = time.time()
    hist, handles = {v: 0 for v in R.VARIANTS}, {v: set() for v in R.VARIANTS}
    strong = []
    modes = (CENTER, CENTER, PRE_PADDED, LEGACY)
    k = 0
    for ci, cfg in enumerate(R.sweep_configs()):
        mel = handle(cfg)
        assert cfg.generic()
        for n in R.clip_lengths(cfg, cfg.sample_rate):
            k += 1
            mode, layout = modes[k % 4], k % 2
            kind = R.SIGNALS[k % len(R.SIGNALS)]
            last = 0.0 if k % 3 else -0.75
            a = R.signal(kind, n, cfg.sample_rate, seed=ci)
            got, T, Tp = run(mel, cfg, a, mode, last, layout)
            want_T = R.frame_count(cfg, n, mode)
            assert T == want_T, (cfg, n, mode, T, want_T)
            if T == 0:
                assert Tp == (0 if mode == LEGACY else 1) and not got.any(), (cfg, n, mode)
                continue
            assert Tp == (T if mode == LEGACY else -(-T // cfg.pad_to) * cfg.pad_to) and not got[T:].any()
            v = cfg.variant(mode)
            hist[v] += 1
            handles[v].add(ci)
            r = restated(mel, cfg, a, mode, last if mode != LEGACY else 0.0, T)
            _note(v, R.compare(got[:T], cfg, r, (cfg, n, mode, layout, kind)))
            if kind in ("noise", "speech"):
                f, m = R.strongest(r, cfg.floor)
                if f.size:
                    _, bL = R.bar(cfg, r)
                    ceil = R.strong_ceiling(cfg, r, (f, m))
                    # below the old 1e-4 bar wherever the strongest band spans <= 16 quads; wider strong bands (1 to 3
                    # mels at large nFFT) carry the fmaf chain's worst case (4 nq + 1)u, which can exceed it
                    assert (bL[f, m] <= ceil).all() and (ceil[r.nq[m] <= 16] < 1e-4).all(), (cfg, n)
                    strong.append(bL[f, m])
    print("\nvariant (reflect, spectrum, affine): calls / handles / worst |d| / bar")
    for v in R.VARIANTS:
        print(f"  {v}: {hist[v]} / {len(handles[v])} / {WORST.get(v, 0.0):.3g}")
    assert all(len(h) >= 3 for h in handles.values()), handles
    s = np.concatenate(strong)
    print(f"log-domain bar at each frame's strongest mel (noise, speech; {s.size} frames): median {np.median(s):.3g}, "
          f"99% {np.quantile(s, 0.99):.3g}, max {s.max():.3g}")
    print(f"variant matrix: {time.time() - t0:.1f} s")


# ================================================================================================ b. Cohere on mel512_kernel
def test_cohere_preset_on_mel512_at_both_precisions(gpu_lib):
    cfg = Cfg.from_ex(ex_config("cohere"))
    assert not cfg.generic()
    for prec, f32t in ((Precision.f64, False), (Precision.f32, True)):
        mel = handle(cfg, prec)
        calls = 0
        for kind in ("noise", "speech", "tone", "square"):
            for n in (1, 255, 256, 257, 160 * 5 + 1, 16000 * 2 + 7):
                for mode in (CENTER, PRE_PADDED, LEGACY):
                    a = R.signal(kind, n, 16000, seed=n)
                    got, T, _ = run(mel, cfg, a, mode, 0.5 if mode != LEGACY else 0.0, (n + mode) % 2)
                    if T == 0:
                        continue
                    r = restated(mel, cfg, a, mode, 0.5 if mode != LEGACY else 0.0, T)
                    _note(f"mel512 {prec.name}", R.compare(got[:T], cfg, r, (prec, kind, n, mode), f32_transform=f32t))
                    calls += 1
        assert calls >= 40
    print(f"\nCohere on mel512_kernel, worst |d| / bar: F64 {WORST['mel512 f64']:.3g}, F32 {WORST['mel512 f32']:.3g}")


# ================================================================================================ c. class entry points
COHERE = [dict(mag_power=1.0), dict(mag_power=1.5), dict(mag_power=2.0), dict(win_length=401), dict(win_length=1000),
          dict(hop_length=161), dict(hop_length=441), dict(n_mels=1), dict(n_mels=64), dict(n_mels=129),
          dict(n_mels=257), dict(f_min=125.0, f_max=3000.0), dict(f_min=20.0, f_max=7000.0), dict(preemph=0.0)]
STYLETTS2 = [dict(n_fft=1024, win_length=1024), dict(n_fft=4096, win_length=2401, hop_length=600),
             dict(win_length=1201, hop_length=301), dict(hop_length=2500), dict(n_mels=1), dict(n_mels=257),
             dict(filter_sample_rate=22050), dict(filter_sample_rate=24000), dict(mean=1.5, std=-0.37)]
LUXTTS = [dict(n_fft=512, win_length=512, hop_length=129), dict(n_fft=2048, win_length=2048), dict(hop_length=255), dict(n_mels=1), dict(n_mels=257),
          dict(sample_rate=16000), dict(sample_rate=48000), dict(log_floor=1e-5), dict(log_floor=1e-10)]


def test_class_entry_points_at_other_parameters(gpu_lib, oracle):
    for v in COHERE:
        coh = CohereMelSpectrogram(CohereMelSpectrogram.Config(**v))
        c = coh.config
        kw = dict(sample_rate=c.sample_rate, win_length=c.win_length, hop_length=c.hop_length, n_mels=c.n_mels,
                  f_min=c.f_min, f_max=c.f_max, preemph=c.preemph, mag_power=c.mag_power)
        for kind in ("speech", "noise", "nan"):
            for n in (1, c.hop_length + 5, 16000 * 3 + 7):
                a = R.signal("noise" if kind == "nan" else kind, n, 16000, seed=n)
                if kind == "nan":
                    a[n // 2] = np.nan
                got, valid = coh.features(a, -1)
                ref, rvalid = OT.cohere_compute(a, **kw)
                assert valid == rvalid == n // c.hop_length and got.shape == ref.shape, (v, n)
                assert not got[:, valid:].any()
                lib_fin, ref_fin = np.isfinite(got[:, :valid]).all(1), np.isfinite(ref[:, :valid]).all(1)
                assert not (~lib_fin & ref_fin).any(), (v, kind, n)
                if valid > 1:
                    # the log-mel budget: the library and the oracle each within the derived bar of the restatement
                    # (with the oracle's two-rounded pre-emphasis in S_f), so at most twice the bar apart
                    cfg = Cfg.from_ex(ex_config("cohere", sample_rate=c.sample_rate, win_length=c.win_length,
                                                hop_length=c.hop_length, n_mels=c.n_mels, n_fft=coh.n_fft,
                                                f_min=c.f_min, f_max=c.f_max, preemph=c.preemph,
                                                spectrum_power=c.mag_power))
                    r = R.restate(cfg, coh.mel.get_hann_window(), coh.mel.get_filterbank(), a, CENTER, 0.0,
                                  1 + n // c.hop_length, preemph_two_roundings=True)
                    _, bL = R.bar(cfg, r)
                    frac, _ = cmvn_frac(coh, a, got, ref, valid, e=2 * bL[:valid])
                    if frac is not None:
                        _note("cohere cmvn", frac)
                        assert frac <= 1.0, (v, kind, n, frac)
    for v in STYLETTS2:
        sty = StyleTTS2MelExtractor(**v)
        cfg = Cfg.from_ex(ex_config("styletts2", **{{"mean": "log_mean", "std": "log_std"}.get(k, k): x
                                                    for k, x in v.items()}))
        for kind in ("speech", "noise"):
            for n in (0, 1, cfg.n_fft // 2, cfg.n_fft // 2 + 1, 5 * cfg.hop + 1, 24000 * 2 + 3):
                a = R.signal(kind, n, 24000, seed=n)
                got, T = sty.compute(a)
                assert T == 1 + n // cfg.hop
                r = restated(sty.mel, cfg, a, CENTER, 0.0, T)
                _note("styletts2", R.compare(got.T, cfg, r, ("styletts2", v, kind, n)))
                ref, rT = OT.styletts2_compute(a, **v)
                assert rT == T
                _note("styletts2 oracle", R.compare(ref.T, cfg, r, ("styletts2 oracle", v, kind, n)))
    for v in LUXTTS:
        mel = AudioMelSpectrogram.from_ex_config(ex_config("luxtts", **v))
        cfg = Cfg.from_ex(ex_config("luxtts", **v))
        L = mel._L
        for kind in ("speech", "noise"):
            for n in (1, cfg.hop // 2, cfg.n_fft // 2 + 1, 5 * cfg.hop + 1, cfg.sample_rate * 2 + 3):
                a = R.signal(kind, n, cfg.sample_rate, seed=n)
                T = (n + cfg.hop // 2) // cfg.hop
                out = np.zeros((max(T, 1), cfg.n_mels), F32)
                fr = C.c_int64()
                _lib.check(L.fa_mel_luxtts_features(mel._h, a.ctypes.data, n, out.ctypes.data, out.size, C.byref(fr)),
                           "fa_mel_luxtts_features")
                assert fr.value == T
                if T == 0:
                    continue
                r = restated(mel, cfg, a, CENTER, 0.0, T)
                _note("luxtts", R.compare(out[:T], cfg, r, ("luxtts", v, kind, n)))
                ref = OT.luxtts_extract(a, n_fft=cfg.n_fft, hop_length=cfg.hop, n_mels=cfg.n_mels,
                                        sample_rate=cfg.sample_rate, log_floor=cfg.floor)
                _note("luxtts oracle", R.compare(ref, cfg, r, ("luxtts oracle", v, kind, n)))
    print("\nclass entry points, worst |d| / bar: " + ", ".join(f"{k} {WORST[k]:.3g}" for k in
                                                              ("cohere cmvn", "styletts2", "styletts2 oracle", "luxtts",
                                                               "luxtts oracle") if k in WORST))


# ================================================================================================ d. CMVN kernel
def test_cohere_cmvn_kernel_bit_for_bit_at_partial_ctas(gpu_lib):
    cases = 0
    for M in (1, 31, 32, 33, 127, 128, 129, 255, 257, 512):
        hop = 40
        coh = CohereMelSpectrogram(CohereMelSpectrogram.Config(n_mels=M, hop_length=hop, win_length=64))
        for valid in (0, 1, 2, 70):
            n = valid * hop + 7
            a = R.signal("speech", n, 16000, seed=M) + F32(1e-3)
            T = 1 + n // hop
            mel, ml, nf = coh.mel._run(a, 0.0, CENTER, T, TIME_MAJOR)
            lm = mel[:T * M].reshape(T, M)
            for W in sorted({1, 31, 32, 33, 65, max(valid - 1, 0), valid, valid + 1}):
                got, fl = coh.features(a, W)
                ref = OT.cohere_cmvn(lm, valid, W)
                assert same_bits(got, ref), (M, valid, W)
                assert fl == min(valid, W)
                cases += 1
    print(f"\ncohere_cmvn_kernel: {cases} cases bit for bit")


# ================================================================================================ e. invariants
def _one_per_variant():
    """The first sweep handle of each (reflect edge, spectrum, affine) kind whose window is not the all-zero length-1
    window; its .center and .prePadded calls launch the generic kernel's 12 variants between them."""
    seen, out = set(), []
    for cfg in R.sweep_configs():
        v = (cfg.reflect, cfg.spectrum, cfg.affine)
        if v not in seen and cfg.win > 1:
            seen.add(v)
            out.append(cfg)
    assert len(out) == 12 and {c.variant(m) for c in out for m in (CENTER, PRE_PADDED)} == set(R.VARIANTS)
    return out


def test_bitwise_invariants_per_variant(gpu_lib):
    rng = np.random.default_rng(3)
    for cfg in _one_per_variant():
        mel = handle(cfg)
        clips = [R.signal("speech", int(m), cfg.sample_rate, seed=i)
                 for i, m in enumerate([1, 2, cfg.n_fft // 2 - 1, cfg.n_fft // 2, 3 * cfg.hop + 5, cfg.sample_rate + 17])]
        clips += [rng.standard_normal(int(rng.integers(3, 20000))).astype(F32) for _ in range(6)]
        last = rng.standard_normal(len(clips)).astype(F32)
        for mode in (CENTER, PRE_PADDED):
            for i, c in enumerate(clips[:6]):
                tm, ml, nf = mel._run(c, float(last[i]), mode, None, TIME_MAJOR)
                mm, ml2, nf2 = mel._run(c, float(last[i]), mode, None, MEL_MAJOR)
                assert (ml, nf) == (ml2, nf2)
                assert same_bits(tm[:nf * cfg.n_mels].reshape(nf, cfg.n_mels).T,
                                 mm[:nf * cfg.n_mels].reshape(cfg.n_mels, nf)), (cfg, i, mode)
            for tmj in (True, False):
                out, oo, ml, nf = mel.compute_batch(clips, last_samples=last, padding_mode=mode, time_major=tmj)
                for i, c in enumerate(clips):
                    single, sml, snf = mel._run(c, float(last[i]), mode, None, TIME_MAJOR if tmj else MEL_MAJOR)
                    assert (ml[i], nf[i]) == (sml, snf) and same_bits(out[oo[i]:oo[i + 1]], single[:snf * cfg.n_mels])
                packed = np.concatenate(clips)
                offs = np.zeros(len(clips) + 1, np.int64)
                offs[1:] = np.cumsum([c.size for c in clips])
                d_in, d_out = _lib.DeviceBuffer(4 * packed.size), _lib.DeviceBuffer(4 * int(oo[-1]))
                d_in.upload(packed)
                bml, bnf = mel.compute_batch_device(d_in, offs, d_out, oo, padding_mode=mode, time_major=tmj)
                _lib.synchronize()   # the device entry points are asynchronous on the handle's stream
                host, _, hml, hnf = mel.compute_batch(clips, padding_mode=mode, time_major=tmj)
                assert np.array_equal(bml, hml) and np.array_equal(bnf, hnf)
                assert same_bits(d_out.download(int(oo[-1]), F32), host[:int(oo[-1])]), (cfg, mode, tmj)
            c = clips[5]
            host, hml, hnf = mel._run(c, float(last[5]), mode, None, TIME_MAJOR)
            d_in, d_out = _lib.DeviceBuffer(4 * c.size), _lib.DeviceBuffer(4 * cfg.n_mels * hnf)
            d_in.upload(c)
            dml, dnf = mel.compute_device(d_in, c.size, d_out, float(last[5]), mode)
            _lib.synchronize()
            assert (dml, dnf) == (hml, hnf) and same_bits(d_out.download(dnf * cfg.n_mels, F32), host[:dnf * cfg.n_mels])


@pytest.mark.parametrize("shape", [dict(n_fft=32, win_length=32, hop_length=7), dict(n_fft=32, win_length=1, hop_length=45),
                                   dict(n_fft=4096, win_length=4095, hop_length=1001),
                                   dict(n_fft=4096, win_length=2049, hop_length=4099)])
def test_pipeline_units_equal_one_unit_on_reflect_handles(gpu_lib, shape):
    cfg = Cfg.from_ex(ex_config("luxtts", n_mels=40, **shape))
    mel = handle(cfg)
    x = R.signal("noise", 4096 * 3 * cfg.hop + 4100, cfg.sample_rate)   # >= 3 units of >= 4096 frames
    T = 1 + x.size // cfg.hop
    outs = []
    for chunks in (1, 2, 7, 24):
        mel._L.fa_mel_set_pipeline_chunks(mel._h, chunks)
        outs.append(run(mel, cfg, x, CENTER, 0.0, TIME_MAJOR, T)[0])
    mel._L.fa_mel_set_pipeline_chunks(mel._h, 24)
    for o in outs[1:]:
        assert same_bits(o, outs[0]), shape
    # the first and last frames against the restatement, the reflections at both ends of a multi-unit clip.  The tail
    # is restated on a suffix that starts q hops in: its right reflection is the clip's, and its first frames, which
    # reflect at the suffix's start, are not compared.
    w, fb = mel.get_hann_window(), mel.get_filterbank()
    R.compare(outs[0][:6], cfg, R.restate(cfg, w, fb, x, CENTER, 0.0, 6), (shape, "head"))
    q = T - 6 - (cfg.n_fft // 2 // cfg.hop + 1)
    r = R.restate(cfg, w, fb, x[q * cfg.hop:], CENTER, 0.0, T - q)
    R.compare(outs[0][T - 6:], cfg, R.Restated(*(getattr(r, f)[-6:] if f in ("out", "L", "E", "S", "R", "absX")
                                                 else getattr(r, f) for f in r.__dataclass_fields__)), (shape, "tail"))


def _units(T, max_units):
    """The unit count of MelPlan::compute_host (unit_bounds): at most max_units, each of at least 4096 frames."""
    K = max(1, min(max_units, T // 4096))
    while K > 1:
        w = [4] * K if K < 6 else [1 if e == 0 else (2 if e == 1 else 4) for e in (min(c, K - 1 - c) for c in range(K))]
        if T * w[0] // sum(w) >= 4096:
            break
        K -= 1
    return K


def test_audio_to_mel_equals_mel_of_the_resampled_pcm(gpu_lib):
    """Converted PCM runs in units of ~10 MiB of input (at most pcm_bytes / 10 MiB + 1) and >= 4096 frames: 170 s of
    48 kHz stereo int16 (32.6 MB) and of 44.1 kHz float (30.0 MB) give 3 units at 24 kHz on both handles, so the reflect
    unit ranges and the resampler's per-unit input windows are crossed.  The launch count confirms the units ran."""
    rng = np.random.default_rng(8)
    for make in (StyleTTS2MelExtractor, LuxTtsMelExtractor):
        mel = make().mel
        conv = AudioConverter(sample_rate=mel.sample_rate)
        st16 = (rng.standard_normal((48000 * 170, 2)) * 3000).astype(np.int16)
        fl = (rng.standard_normal(44100 * 170) * 0.3).astype(F32)
        short = (rng.standard_normal((20, 2)) * 3000).astype(np.int16)                   # <= nFFT/2 after conversion
        for pcm, rate, ch, inter in ((st16, 48000, 2, True), (fl, 44100, 1, False), (short, 48000, 2, True)):
            mono = conv.resample_buffer(pcm, rate, channels=ch, interleaved=inter)
            want, wml, wnf = mel._run(mono, 0.0, CENTER, None, TIME_MAJOR)
            launches = {}
            for chunks in (1, 2, 7, 24):
                mel._L.fa_mel_set_pipeline_chunks(mel._h, chunks)
                before = _lib.kernel_launch_count()
                got, ml, nf, rs = mel.compute_from_pcm(pcm, rate, channels=ch, interleaved=inter)
                launches[chunks] = _lib.kernel_launch_count() - before
                assert rs == mono.size and (ml, nf) == (wml, wnf)
                assert same_bits(got, want[:nf * mel.n_mels]), (make.__name__, rate, chunks)
            mel._L.fa_mel_set_pipeline_chunks(mel._h, 24)
            if pcm is short:
                assert mono.size <= mel.n_fft // 2
                continue
            units = {c: _units(wml, min(c, pcm.nbytes // (10 << 20) + 1)) for c in launches}
            assert units[1] == 1 and units[2] == 2 and units[7] == units[24] == 3, units
            for c in (2, 7, 24):
                assert launches[c] > launches[1], (make.__name__, rate, launches)


# ================================================================================================ f. non-finite input
def _reads(cfg, n, T, mode, k):
    """Frames whose in-window samples read sample k: directly, through a reflection, or as pre-emphasis's x[i-1]."""
    off = 0 if mode == LEGACY else (cfg.n_fft - cfg.win) // 2
    pad = cfg.n_fft // 2 if mode == CENTER else 0
    pre = cfg.preemph != 0.0 and mode != LEGACY
    hit = np.zeros(T, bool)
    j = off + np.arange(cfg.win)
    for f in range(T):
        i = f * cfg.hop - pad + j
        if cfg.reflect and mode == CENTER:
            src = R.reflect_clamped(i, n)
        else:
            src = i[(i >= 0) & (i < n)]
        hit[f] = (src == k).any() or (pre and (src == k + 1).any())
    return hit


def test_nan_footprint_for_every_variant(gpu_lib):
    for cfg in _one_per_variant():
        mel = handle(cfg)
        fb = mel.get_filterbank()
        live = fb.any(1)
        n = 6 * cfg.hop + cfg.n_fft
        for mode in (CENTER, PRE_PADDED):
            for k in (0, 1, cfg.n_fft // 2, n // 2, n - 1):
                a = R.signal("noise", n, cfg.sample_rate)
                a[k] = np.nan
                got, T, _ = run(mel, cfg, a, mode, 0.25)
                hit = _reads(cfg, n, T, mode, k)
                assert not np.isnan(got[:T][~hit]).any(), (cfg, mode, k)   # log floor 0 makes silent mels -inf
                assert np.isnan(got[:T][hit][:, live]).all(), (cfg, mode, k)
                assert not np.isnan(got[:T][hit][:, ~live]).any(), (cfg, mode, k)


def test_overflow_footprint_is_the_class_oracles(gpu_lib):
    """A sample of 3e38 overflows the float32 power (|X| above sqrt(FLT_MAX) ~ 1.8e19 squares to inf); the kernels
    square before sqrtf, so for |X| and |X|^p the magnitude is inf there too, like the reference classes' sqrtf(re^2 +
    im^2), and the log-mel is inf in every band that holds such a bin.  The library is non-finite only where the class
    oracle is (DESIGN §2)."""
    for v in ({}, dict(n_fft=1024, win_length=1024, hop_length=301), dict(n_mels=257)):
        sty = StyleTTS2MelExtractor(**v)
        for n in (5000, 700):
            a = R.signal("noise", n, 24000)
            a[n // 3] = F32(3e38)
            got, _ = sty.compute(a)
            ref, _ = OT.styletts2_compute(a, **v)
            assert not (~np.isfinite(got) & np.isfinite(ref)).any() and (~np.isfinite(got)).any(), v
    for v in ({}, dict(n_fft=512, win_length=512, hop_length=129)):
        lux = AudioMelSpectrogram.from_ex_config(ex_config("luxtts", **v))
        for n in (5000, 700):
            a = R.signal("noise", n, 24000)
            a[n // 3] = F32(3e38)
            ext = LuxTtsMelExtractor()
            ext.mel, ext.hop_length, ext.n_mels = lux, lux.hop_length, lux.n_mels
            got = ext.extract(a)
            ref = OT.luxtts_extract(a, n_fft=lux.n_fft, hop_length=lux.hop_length)
            assert not (~np.isfinite(got) & np.isfinite(ref)).any() and (~np.isfinite(got)).any(), v
    for mp in (1.0, 1.5, 2.0):
        coh = CohereMelSpectrogram(CohereMelSpectrogram.Config(mag_power=mp, preemph=0.0))
        a = R.signal("noise", 16000, 16000)
        a[5000] = F32(3e38)
        got, valid = coh.features(a, -1)
        ref, _ = OT.cohere_compute(a, mag_power=mp, preemph=0.0)
        lib_bad, ref_bad = ~np.isfinite(got[:, :valid]).all(1), ~np.isfinite(ref[:, :valid]).all(1)
        assert not (lib_bad & ~ref_bad).any() and lib_bad.any(), mp


def test_zz_report_runtime():
    print(f"\ntest_gpu_mel_ex_sweep.py: {time.time() - T0:.1f} s; worst |d| / bar: "
          + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items(), key=str)))
