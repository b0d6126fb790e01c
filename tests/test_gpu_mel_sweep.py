"""Log-mel kernels against the oracle across their configuration space (run with ``-m gpu`` on an H100).

``AudioMelSpectrogram`` takes any nFFT, hop, window length, mel count, sample rate, log floor and padTo; the library
dispatches them to ``mel512_kernel<double>``, ``mel512_kernel<f32x2>`` (nFFT 512, even hop, shared memory permitting) and
``mel_generic_kernel`` (everything else).  This file sweeps those axes through the C ABI, checks the invariants that must hold
bit for bit between entry points, and feeds non-finite input.

Bars (DESIGN §4.1): FP64 transform and the generic kernel |d| <= 1e-5 + 4e-7 |ref| (the second term: 2 ulp of the device log
at large magnitudes, e.g. log floor 0).  Float32 pairs 1e-4, widened only for mel values more than 12 nats below their frame's
strongest one, where the float32 transform's own rounding noise is what is compared (DESIGN §2; the lane emulator in
test_host_logic.py shows the same values on the CPU).  Frames whose window holds a NaN are NaN in every mel whose band is
non-empty; the oracle multiplies by the dense filterbank and is NaN in every mel (DESIGN §2, stated deviation).
"""
import numpy as np
import pytest

from fluidaudio_b200 import _lib, synth
from fluidaudio_b200.mel import AudioMelSpectrogram, LSEENDMelFrontend, PaddingMode, Precision

pytestmark = pytest.mark.gpu

FRAMES = (1, 2, 15, 16, 17, 31, 33)                 # tile edges (16 frames) and odd frame pairs
WINS = (512, 449, 448, 400, 385, 384, 383, 256, 64)  # both sides of the mid_full boundary (buffer positions [64, 448))
MELS = (1, 3, 23, 40, 81, 128, 200, 257)
RATES = (16000, 8000, 22050, 48000)
FLOORS = (2.0 ** -24, 1e-10, 1e-38, 0.0)            # 1e-38 is subnormal: the kernel's __log2f path
EVEN_HOPS = (160, 2, 64, 128, 158, 256, 320, 512, 514, 1000)
CENTER, PRE_PADDED, LEGACY = 0, 1, 2
TIME_MAJOR, MEL_MAJOR = 0, 1

WORST = {}                                          # largest |d| seen per kernel, reported in every failure message


def fp64_bar(r, top):
    return 1e-5 + 4e-7 * np.abs(r)


def f32_bar(r, top):
    # 1e-4, growing with the depth below the frame's strongest mel past 12 nats, capped at 2e-3: twice the largest
    # float32-pair deviation measured over this file (9.8e-4; the lane emulator's largest is 5.1e-4)
    return np.minimum(2e-3, 1e-4 * np.maximum(1.0, np.exp(top - r - 12.0)))


_PROBE = None


def plan_kernel(m):
    """Which kernel the plan runs.  mel_generic_kernel ignores the precision switch (FP64 transform either way), so its two
    settings agree bit for bit; the specialised kernel's FP64 and float32 transforms never do on 101 frames of noise."""
    global _PROBE
    if _PROBE is None:
        _PROBE = synth.tone_noise_audio(16000, seed=1)
    prec = m.precision
    outs = []
    for p in (Precision.f64, Precision.f32):
        m.set_precision(p)
        outs.append(m.compute_flat_transposed(_PROBE)[0].copy())
    m.set_precision(prec)
    return "generic" if np.array_equal(outs[0], outs[1]) else "mel512"


def kernel_of(kind, precision):
    return (kind, "f32" if kind == "mel512" and precision == Precision.f32 else "f64")


def bar_of(kernel):
    return f32_bar if kernel[1] == "f32" else fp64_bar


def compare(got, ref, fb, bar, kernel, what):
    """got, ref: [frames x nMels].  NaN frames of the oracle are NaN in every non-empty band, other frames finite where the
    oracle is finite, equal where it is not (log 0 = -inf), and within the bar."""
    got = np.asarray(got, np.float32)
    ref = np.asarray(ref, np.float32)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    nan_rows = np.isnan(ref).any(axis=1)
    band = fb.any(axis=1)
    assert np.isnan(got[nan_rows][:, band]).all(), (what, "NaN frame lost its NaN")
    g, r = got[~nan_rows], ref[~nan_rows]
    fin = np.isfinite(r)
    assert np.array_equal(g[~fin], r[~fin]), (what, "non-finite values differ")
    assert np.isfinite(g[fin]).all(), (what, "non-finite value where the oracle is finite")
    if fin.any():
        top = np.broadcast_to(np.where(fin, r, -np.inf).max(axis=1, keepdims=True), r.shape)
        d = np.abs(g[fin] - r[fin])
        key = " ".join(kernel)
        WORST[key] = max(WORST.get(key, 0.0), float(d.max()))
        bad = d > bar(r[fin], top[fin])
        assert not bad.any(), (what, "max |d|", float(d.max()), "largest per kernel", dict(WORST))
    return nan_rows


def length_for(frames, hop, win, n_fft=512):
    """A sample count whose .center frame count is about `frames`."""
    return max(1, (frames - 1) * hop + win - n_fft + 1)


def oracle_run(oracle, cfg, x, last, mode, expected=None):
    """[frames x nMels] reference, melLength, numFrames in the library's mode numbering."""
    if mode == LEGACY:
        ref, T = oracle.mel_legacy(cfg, x)
        return (ref.T if T else np.zeros((0, cfg.n_mels), np.float32)), T, T
    ref, ml, nf = oracle.mel_flat_transposed(cfg, x, last=last, padding_mode=mode, expected_frames=expected)
    return ref.reshape(nf, cfg.n_mels), ml, nf


# ================================================================================================ exhaustive axes
def test_every_even_hop_both_precisions(gpu_lib, oracle):
    """Every even hop 2..1024 against the oracle, one short clip each: the specialised kernel while its shared memory fits,
    the generic kernel past it, no hop rejected.  At 80 mels on H100 (227 KB per block) the switch lies near hop 890."""
    fb = oracle.mel_filterbank(512, 80)
    kinds = {}
    for hop in range(2, 1025, 2):
        x = synth.tone_noise_audio(length_for(FRAMES[hop // 2 % 7], hop, 400), seed=hop)
        m = AudioMelSpectrogram(n_mels=80, hop_length=hop)
        kinds[hop] = kind = plan_kernel(m)
        ref, rml, rnf = oracle_run(oracle, oracle.mel_config(n_mels=80, hop_length=hop), x, 0.1, CENTER)
        for prec in (Precision.f64, Precision.f32):
            m.set_precision(prec)
            got, ml, nf = m.compute_flat_transposed(x, last_audio_sample=0.1)
            assert (ml, nf) == (rml, rnf), hop
            k = kernel_of(kind, prec)
            compare(got.reshape(nf, 80), ref, fb, bar_of(k), k, dict(hop=hop, kernel=kind))
        m.close()
    assert all(kinds[h] == "mel512" for h in range(2, 861, 2)), [h for h in range(2, 861, 2) if kinds[h] != "mel512"]
    assert all(kinds[h] == "generic" for h in range(920, 1025, 2)), [h for h in range(920, 1025, 2) if kinds[h] != "generic"]


def test_every_mel_count_both_precisions(gpu_lib, oracle):
    """n_mels 1..512 at hop 160, 16 and 48 kHz: the n_mels + 1 and n_mels + 4 copy-outs, the slot schedule at every group
    count, and the empty filters (from 193 mels at 16 kHz, from 87 at 48 kHz)."""
    for sr in (16000, 48000):
        for nm in range(1, 513):
            fb = oracle.mel_filterbank(512, nm, sr)
            if nm == 512:
                assert not fb.any(axis=1).all(), sr                  # the lowest filters are empty: covered
            x = synth.tone_noise_audio(length_for(FRAMES[nm % 7] + 16 * (nm % 3), 160, 400), seed=nm)
            m = AudioMelSpectrogram(sample_rate=sr, n_mels=nm)
            assert plan_kernel(m) == "mel512", (sr, nm)
            ref, rml, rnf = oracle_run(oracle, oracle.mel_config(sample_rate=sr, n_mels=nm), x, -0.2, CENTER)
            for prec in (Precision.f64, Precision.f32):
                m.set_precision(prec)
                got, ml, nf = m.compute_flat_transposed(x, last_audio_sample=-0.2)
                assert (ml, nf) == (rml, rnf)
                k = kernel_of("mel512", prec)
                compare(got.reshape(nf, nm), ref, fb, bar_of(k), k, dict(sr=sr, n_mels=nm))
            m.close()


# ================================================================================================ cross product
def _run_config(oracle, kw, seed, speech=False):
    """Every mode (centre, prePadded with and without an expected frame count, legacy) in both layouts and both precisions
    against the oracle; mel-major must be the transpose of time-major bit for bit."""
    n_fft, hop, win, nm = kw.get("n_fft", 512), kw["hop_length"], kw["win_length"], kw["n_mels"]
    m = AudioMelSpectrogram(**kw)
    kind = plan_kernel(m)
    if n_fft != 512 or hop % 2 or hop > 1024:
        assert kind == "generic", kw
    cfg = oracle.mel_config(**kw)
    fb = oracle.mel_filterbank(n_fft, nm, kw.get("sample_rate", 16000))
    frames = FRAMES[seed % 7] if seed % 5 else 200 + seed % 37                   # a few hundred frames now and then
    n = max(length_for(frames, hop, win, n_fft), n_fft + 1)
    x = synth.speech_like_audio(n, seed=seed) if speech else synth.tone_noise_audio(n, seed=seed)
    computed = m.frame_count(n, PRE_PADDED)
    calls = [(CENTER, None), (PRE_PADDED, None), (PRE_PADDED, max(1, computed + (3 if seed % 2 else -1))), (LEGACY, None)]
    for mode, expected in calls:
        ref, rml, rnf = oracle_run(oracle, cfg, x, 0.25, mode, expected)
        for prec in (Precision.f64, Precision.f32):
            m.set_precision(prec)
            k = kernel_of(kind, prec)
            bar = bar_of(k)
            if mode == LEGACY and speech and k[1] == "f32":       # no pre-emphasis on the 60 dB fixture (DESIGN §4.1)
                bar = lambda r, top: np.maximum(3e-4, f32_bar(r, top))
            what = dict(kw, mode=mode, expected=expected, precision=int(prec), frames=rnf, speech=speech, kernel=kind)
            tm, ml, nf = m._run(x, 0.25, mode, expected, TIME_MAJOR)
            assert (ml, nf) == (rml, rnf), what
            tm = tm[: nf * nm].reshape(nf, nm)
            compare(tm, ref, fb, bar, k, what)
            mm, ml2, nf2 = m._run(x, 0.25, mode, expected, MEL_MAJOR)
            assert (ml2, nf2) == (ml, nf) and np.array_equal(mm[: nf * nm].reshape(nm, nf), tm.T), what
    m.close()


def test_configuration_cross_product(gpu_lib, oracle):
    """Window length x sample rate x floor mode x log floor on the specialised kernel (both window placements: centred
    for .center / .prePadded, offset 0 for compute()), with the hop, mel count and padTo dealt round-robin."""
    i = 0
    for win in WINS:
        for sr in RATES:
            for clamped in (0, 1):
                for fl in FLOORS:
                    i += 1
                    kw = dict(sample_rate=sr, n_mels=MELS[i % len(MELS)], hop_length=EVEN_HOPS[i % len(EVEN_HOPS)],
                              win_length=win, pad_to=(1, 3, 16)[i % 3], log_floor=fl, log_floor_mode=clamped)
                    _run_config(oracle, kw, i, speech=i % 4 == 0)


def test_generic_kernel_configurations(gpu_lib, oracle):
    """nFFT 64 / 256 / 1024 / 4096, odd hops, hops longer than nFFT, and nFFT 512 configurations the specialised kernel does
    not take, in both floor modes and every log floor."""
    cases = [(64, 64, 17, 10), (64, 48, 1025, 8), (256, 200, 80, 23), (256, 256, 3, 40), (1024, 800, 320, 80),
             (1024, 1000, 1025, 128), (4096, 4096, 4097, 257), (4096, 2000, 511, 81), (512, 400, 161, 80),
             (512, 385, 1025, 3), (512, 512, 1026, 200)]
    i = 0
    for n_fft, win, hop, nm in cases:
        for clamped in (0, 1):
            for fl in FLOORS:
                i += 1
                kw = dict(sample_rate=RATES[i % 4], n_fft=n_fft, n_mels=nm, hop_length=hop, win_length=win,
                          pad_to=(1, 3, 16)[i % 3], log_floor=fl, log_floor_mode=clamped, window_periodic=bool(i % 2))
                _run_config(oracle, kw, i, speech=i % 3 == 0)


# ================================================================================================ bitwise invariants
class _View:
    """A device pointer at a byte offset inside a DeviceBuffer."""

    def __init__(self, buf, byte_offset):
        import ctypes as C
        self.ptr = C.c_void_p(buf.ptr.value + byte_offset)
        self.nbytes = buf.nbytes - byte_offset


KERNEL_CONFIGS = [dict(n_mels=80), dict(n_mels=81, hop_length=158, win_length=383),
                  dict(n_mels=23, n_fft=256, hop_length=80, win_length=200), dict(n_mels=80, hop_length=161)]
CTAS_PER_SM = 2       # both kernels launch at most 2 CTAs per SM here (mel512: kCtasPerSm; generic: 16 / 8 warps per CTA)
BATCH_GROUPS = 32     # compute_batch cuts a batch into up to 32 launches


def _tiny_clip_batch(m, hop, win, n_fft, grid):
    """Clips of 1..33 frames, BATCH_GROUPS x (2 grid + 1) of them: every compute_batch launch, and the one
    compute_batch_device launch, hold more than two tiles per CTA, so each CTA hands over between units (TileInfo slots,
    the next clip's bulk copy, a new `last`).  Slices of one signal at odd offsets and lengths."""
    per_group = 2 * grid + 1
    count = BATCH_GROUPS * per_group
    frames = 1 + (np.arange(count) * 7) % 33
    lens = np.array([length_for(int(f), hop, win, n_fft) for f in frames], np.int64) + np.arange(count) % 5
    base = synth.tone_noise_audio(1 << 20, seed=21)
    starts = (np.arange(count, dtype=np.int64) * 7919) % (base.size - int(lens.max()))
    offsets = np.zeros(count + 1, np.int64)
    offsets[1:] = np.cumsum(lens)
    packed = np.concatenate([base[st:st + n] for st, n in zip(starts, lens)])
    tiles = np.array([-(-m.frame_count(int(n)) // 16) for n in lens])
    for g in range(BATCH_GROUPS):
        assert tiles[g * per_group:(g + 1) * per_group].sum() > 2 * grid, g
    last = np.linspace(-0.3, 0.3, count).astype(np.float32)
    return packed, offsets, last, per_group


@pytest.mark.parametrize("kw", KERNEL_CONFIGS, ids=["mel512_80", "mel512_81", "generic_256", "generic_odd_hop"])
def test_entry_points_agree_bitwise(gpu_lib, kw):
    """For each kernel and precision: batch == one by one with thousands of tiny clips (more than two tiles per CTA, so
    tiles of different units follow each other in one CTA), compute_batch_device == compute_batch, device == host, input
    at +4 bytes (no bulk copy) == aligned input, output at +4 bytes == aligned output (compute_device, compute_batch_device
    with odd out_offsets, zero-copy into pinned memory at +1 float with several pipeline units), and no float outside a
    clip's rows written; mel-major == transpose of time-major."""
    import torch
    grid = CTAS_PER_SM * torch.cuda.get_device_properties(0).multi_processor_count
    nm = kw["n_mels"]
    hop, win, n_fft = kw.get("hop_length", 160), kw.get("win_length", 400), kw.get("n_fft", 512)
    for prec in (Precision.f64, Precision.f32):
        m = AudioMelSpectrogram(precision=prec, **kw)
        packed, offsets, last, per_group = _tiny_clip_batch(m, hop, win, n_fft, grid)
        count = offsets.size - 1
        out, offs, ml, nf = m.compute_batch(None, last_samples=last, packed_audio=packed, offsets=offsets)
        # one by one: the whole first launch of compute_batch, then every 53rd clip
        for i in list(range(per_group)) + list(range(per_group, count, 53)):
            a = packed[offsets[i]:offsets[i + 1]]
            single = m.compute_flat_transposed(a, last_audio_sample=float(last[i]))[0]
            assert np.array_equal(out[offs[i]:offs[i + 1]], single), (prec, i)
        # the same batch from HBM in ONE launch: clips at odd sample offsets, outputs at odd float offsets (+ one gap
        # float each); every float the kernel must not write keeps its sentinel
        sizes = np.diff(offs)
        d_a = _lib.DeviceBuffer(packed.nbytes + 64)
        d_a.upload(packed)
        for shift in (0, 1):
            out_off = offs + shift * (np.arange(count + 1) + 1)
            total = int(out_off[-1]) + 8
            d_o = _lib.DeviceBuffer(total * 4)
            d_o.upload(np.full(total, 7.0, np.float32))
            ml2, nf2 = np.zeros(count, np.int64), np.zeros(count, np.int64)
            _lib.check(m._L.fa_mel_compute_batch_device(m._h, d_a.ptr, offsets.ctypes.data, count, last.ctypes.data,
                                                        CENTER, TIME_MAJOR, d_o.ptr, out_off.ctypes.data, ml2.ctypes.data,
                                                        nf2.ctypes.data), "fa_mel_compute_batch_device")
            _lib.synchronize()
            assert np.array_equal(ml2, ml) and np.array_equal(nf2, nf)
            want = np.full(total, 7.0, np.float32)
            want[np.arange(int(offs[-1])) + np.repeat(shift * (np.arange(count) + 1), sizes)] = out
            assert np.array_equal(d_o.download((total,), np.float32), want), (prec, shift)
            d_o.free()
        d_a.free()
        # device == host, aligned and shifted input, aligned and shifted output, both layouts, nothing written around it
        a = synth.tone_noise_audio(16000 + 37, seed=10)
        T = m.frame_count(a.size)
        host_tm = m.compute_flat_transposed(a)[0]
        host_mm = m.compute_flat(a)[0]
        assert np.array_equal(host_mm.reshape(nm, T), host_tm.reshape(T, nm).T)
        for in_shift in (0, 4):
            d_in = _lib.DeviceBuffer(a.nbytes + 64)
            d_in.upload(np.concatenate([np.zeros(in_shift // 4, np.float32), a]))
            for out_shift in (0, 4):
                d_out = _lib.DeviceBuffer(T * nm * 4 + 64)
                for tm_, host in ((True, host_tm), (False, host_mm)):
                    d_out.upload(np.full(T * nm + 16, 7.0, np.float32))
                    assert m.compute_device(_View(d_in, in_shift), a.size, _View(d_out, out_shift), time_major=tm_) == (T, T)
                    _lib.synchronize()
                    want = np.full(T * nm + 16, 7.0, np.float32)
                    want[out_shift // 4:out_shift // 4 + T * nm] = host
                    assert np.array_equal(d_out.download((T * nm + 16,), np.float32), want), (prec, in_shift, out_shift, tm_)
                d_out.free()
            d_in.free()
        # zero-copy output into pinned memory at +1 float, several pipeline units (the kernel stores into the caller's buffer)
        n = 16000 * 100
        b = synth.tone_noise_audio(n, seed=3)
        T = m.frame_count(n)
        ref = m.compute_flat_transposed(b)[0]
        pin = _lib.PinnedArray(T * nm + 4, np.float32)
        _lib.check(m._L.fa_mel_set_zero_copy_output(m._h, 1), "zero copy")
        _lib.check(m._L.fa_mel_set_pipeline_chunks(m._h, 4), "chunks")
        for shift in (0, 1):
            pin.array[:] = -1.0
            got = m.compute_flat_transposed(b, out=pin.array[shift:shift + T * nm])[0]
            assert np.array_equal(got, ref), (prec, shift)
            assert (pin.array[:shift] == -1.0).all() and (pin.array[shift + T * nm:] == -1.0).all(), (prec, shift)
        pin.free()
        m.close()


# ================================================================================================ non-finite input
def test_nan_samples_poison_exactly_their_frames(gpu_lib, oracle):
    """A NaN inside a frame's window (after pre-emphasis) makes that frame NaN in every non-empty band, in both floor modes;
    one just outside the window leaves the frame finite: the kernels select the in-window samples instead of multiplying
    the whole nFFT buffer by a zero-padded window (NaN * 0 = NaN).  Every window placement; the other frame of a float32
    pair stays finite and within the bar."""
    hop, nm = 160, 40
    for win in WINS:
        for mode in (CENTER, LEGACY):
            off, pad = (0, 0) if mode == LEGACY else ((512 - win) // 2, 256)
            for clamped in (0, 1):
                kw = dict(n_mels=nm, hop_length=hop, win_length=win, log_floor=1e-10, log_floor_mode=clamped)
                m = AudioMelSpectrogram(**kw)
                kind = plan_kernel(m)
                cfg = oracle.mel_config(**kw)
                fb = oracle.mel_filterbank(512, nm)
                for f in (5, 22):                                   # frames in the first and the second tile
                    for j, inside in ((off, True), (off + win - 1, True), (off - 2, False), (off + win, False)):
                        if not 0 <= j < 512:
                            continue
                        x = synth.tone_noise_audio(40 * hop + 512, seed=win + j + f)
                        x[f * hop + j - pad] = np.nan
                        ref, rml, rnf = oracle_run(oracle, cfg, x, 0.0, mode)
                        for prec in (Precision.f64, Precision.f32):
                            m.set_precision(prec)
                            k = kernel_of(kind, prec)
                            got, ml, nf = m._run(x, 0.0, mode, None, TIME_MAJOR)
                            what = dict(kw, mode=mode, f=f, j=j, precision=int(prec))
                            nan_rows = compare(got[: nf * nm].reshape(nf, nm), ref, fb, bar_of(k), k, what)
                            assert nan_rows[f] == inside, what
                m.close()


def test_overflowing_power_is_non_finite_in_the_same_frames(gpu_lib, oracle):
    """|X|^2 beyond float32 range: both sides agree on which frames hold a non-finite value (which mels of such a frame are
    non-finite can differ: the oracle's dense filterbank makes 0 * inf = NaN in every mel, DESIGN §2)."""
    x = synth.tone_noise_audio(16000 * 2, seed=9)
    x[6000:9000] *= np.float32(1e25)
    x[20000:20001] *= np.float32(1e30)
    for kw in (dict(n_mels=80), dict(n_mels=80, log_floor_mode=1, log_floor=1e-10), dict(n_mels=40, n_fft=1024, win_length=800)):
        m = AudioMelSpectrogram(**kw)
        kind = plan_kernel(m)
        ref, _, nf = oracle_run(oracle, oracle.mel_config(**kw), x, 0.0, CENTER)
        bad = ~np.isfinite(ref).all(axis=1)
        assert 0 < bad.sum() < nf
        for prec in (Precision.f64, Precision.f32):
            m.set_precision(prec)
            got = m.compute_flat_transposed(x)[0].reshape(nf, kw["n_mels"])
            assert np.array_equal(~np.isfinite(got).all(axis=1), bad), (kw, prec)
            fine = ~bad
            k = kernel_of(kind, prec)
            compare(got[fine], ref[fine], oracle.mel_filterbank(kw.get("n_fft", 512), kw["n_mels"]), bar_of(k), k, kw)
        m.close()


def test_lseend_nan_chunk_poisons_the_running_mean(gpu_lib, oracle):
    """LS-EEND front end (clamped floor): a NaN sample makes its frames NaN, and the cumulative mean NaN, as in the oracle."""
    a = synth.speech_like_audio(16000 * 3)
    fe = LSEENDMelFrontend()
    cfg = oracle.lseend_config()
    mean, count = np.zeros(23, np.float32), 0
    for n, nan_at in ((8000, None), (8000 + 352, 4000), (4000, None)):
        chunk = a[:n].copy()
        if nan_at is not None:
            chunk[nan_at] = np.nan
        got = fe.process(chunk)
        ref, mean, count = oracle.lseend_features(cfg, chunk, mean, count)
        assert got.shape == ref.shape and fe.cmn_count == count
        assert np.array_equal(np.isnan(got), np.isnan(ref))
        assert np.array_equal(np.isnan(fe.cmn_mean), np.isnan(mean))
        fin = np.isfinite(ref)
        assert np.all(np.abs(got[fin] - ref[fin]) < 1e-4)
    assert np.isnan(fe.cmn_mean).all()
