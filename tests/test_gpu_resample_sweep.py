"""The converter stage (``resample_kernels.cu``) against the oracle across its configuration space (run with ``-m gpu``).

``fa_audio_resample`` / ``fa_audio_to_mel`` take any pair of rates on the 1/1000 Hz grid, 1 to 64 channels, float32 or
int16, planar or interleaved, and run ``mixdown_kernel`` (same rate), ``linear_kernel`` (> 2 channels, or forced) or
``sinc_kernel`` (exact phases when L <= 2048, 1024 interpolated phases otherwise; 32-bit or 64-bit phase arithmetic).

Sinc bar, per output i: |GPU - oracle| <= (taps/4 + 6) 2^-24 S_i, S_i = sum_k A_k |x_k| (``oracle.sinc_resample``:
A_k = |g_k|, or |g_{p,k}| + |g_{p+1,k}| where two rows are blended).  With u = 2^-24, relative to S_i:
  * each of the four accumulators is a chain of at most ceil(taps/4) FMAs, one rounding each: ceil(taps/4) u;
  * the two final adds: 2 u;
  * the float32 table: every coefficient within u of its float64 row value: u;
  * interpolated rows: c1 - c0 and the blending FMA round once each: 2 u (the A_k above covers both rows);
  * the oracle's own float32 result: u / 2.
That sums to ceil(taps/4) + 5.5 <= taps/4 + 6 (taps is even), plus second-order terms.  The worst deviation / bar seen is
reported in every failure message (``WORST``).  Linear is compared bit for bit, NaN masks apart from payloads.
"""
import time

import numpy as np
import pytest

from fluidaudio_b200 import _lib
from fluidaudio_b200.audio_converter import Algorithm, AudioConverter
from fluidaudio_b200.mel import AudioMelSpectrogram, PaddingMode

pytestmark = pytest.mark.gpu

INT_RATES = (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000)
FRACTIONAL = (16001, 44100.5, 47999.99, 8000.1, 22050.25, 11025.001, 44100.001, 48000.001)
TARGETS = (8000, 22050, 44100, 48000)
U = 2.0 ** -24
SMEM_BOUND = 200 * 1024       # make_design: (255 M / L + taps + 8) floats
SMEM_OPT_IN = 48 * 1024       # launches above this ask for the dynamic shared-memory opt-in

WORST = {"ratio": 0.0, "case": None}
_CONV = {}


def conv(out_rate=16000, algorithm=Algorithm.auto):
    key = (float(out_rate), int(algorithm))
    if key not in _CONV:
        _CONV[key] = AudioConverter(sample_rate=out_rate, algorithm=algorithm)
    return _CONV[key]


def noise(channels, frames, seed):
    """planar [channels x frames] float32: full-scale noise plus a tone, so that both large and small taps matter"""
    rng = np.random.default_rng(seed)
    t = np.arange(frames)
    x = 0.7 * rng.uniform(-1, 1, (channels, frames)) + 0.3 * np.sin(2 * np.pi * 0.01 * (1 + np.arange(channels))[:, None] * t)
    return x.astype(np.float32)


def frames_for(count, rin, rout):
    """input frames whose output count (Int(n / (in / out))) is exactly `count`, None when upsampling skips it"""
    n = int(np.ceil(count * rin / rout))
    while n > 0 and int(float(n) / (rin / rout)) > count:
        n -= 1
    while int(float(n) / (rin / rout)) < count:
        n += 1
    return n if int(float(n) / (rin / rout)) == count else None


def check_sinc(oracle, got, mono, rin, rout, what):
    """got vs the oracle's float64 filter within the derived bar; outputs with S_i = 0 must be exactly 0"""
    ref, mag = oracle.sinc_resample(mono, rin, rout, with_magnitude=True)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    if not got.size:
        return
    taps = 2 * oracle.sinc_design(rin, rout).half
    bar = (taps / 4 + 6) * U * mag
    d = np.abs(got.astype(np.float64) - ref.astype(np.float64))
    assert np.isfinite(got).all(), what
    ratio = np.where(bar > 0, d / np.where(bar > 0, bar, 1.0), np.where(d > 0, np.inf, 0.0))
    r = float(ratio.max())
    if r > WORST["ratio"]:
        WORST.update(ratio=r, case=what)
    assert r <= 1.0, (what, "worst output", int(ratio.argmax()), r, "largest so far", WORST)


def same_bits(a, b, what):
    """bitwise equality; NaN only needs to be NaN at the same place (x86 and CUDA payloads differ)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    na, nb = np.isnan(a), np.isnan(b)
    assert np.array_equal(na, nb), (what, "NaN mask")
    assert np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32)), (what, "bits")


def footprint(oracle, rin, rout, count, m):
    """outputs whose 2H-tap window n0 - H + 1 .. n0 + H holds input m"""
    d = oracle.sinc_design(rin, rout)
    n0, _ = oracle.sinc_positions(count, d.L, d.M)
    return (n0 - d.half + 1 <= m) & (m <= n0 + d.half)


# ------------------------------------------------------------------------------------------------ values vs the oracle
def test_sinc_values_integer_and_fractional_rates(gpu_lib, oracle):
    """Every integer rate to 16 kHz (mono float32 planar, stereo int16 interleaved), every integer rate to 8 / 22.05 /
    44.1 / 48 kHz (decimation, upsampling, L > 1), and the interpolated path including the rates whose phases overflow 32
    bits (44100.001, 48000.001 Hz: 64-bit phase arithmetic)."""
    for k, rin in enumerate(INT_RATES + FRACTIONAL):
        n = int(rin * 0.3)
        x = noise(2, n, seed=k)
        if rin != 16000:
            check_sinc(oracle, conv().resample(x[0], rin), x[0], rin, 16000, ("mono", rin))
        i16 = np.round(x * 32767).astype(np.int16)
        i16[0, 5], i16[1, 9] = -32768, 32767
        got = conv().resample_buffer(np.ascontiguousarray(i16.T), rin, interleaved=True)
        if rin == 16000:
            same_bits(got, oracle.mixdown(i16), ("mixdown", rin))
        else:
            check_sinc(oracle, got, oracle.mixdown(i16), rin, 16000, ("stereo int16", rin))
    for k, rin in enumerate(INT_RATES):
        for rout in TARGETS:
            if rin == rout:
                continue
            x = noise(1, int(rin * 0.15), seed=100 + k)[0]
            check_sinc(oracle, conv(rout).resample(x, rin), x, rin, rout, ("to", rin, rout))
    print("worst deviation / bar:", WORST)


def test_sinc_shared_memory_boundaries_and_rejections(gpu_lib, oracle):
    """Integer decimation ratios r at 16 kHz: the last r below the 48 KB dynamic shared-memory opt-in and the first above
    it, and the largest ratio make_design accepts, all derived from its formulas; the next ratio, off-grid rates and rates
    whose reduced terms reach 2^32 return FA_UNSUPPORTED."""
    def launch_bytes(r):        # sinc_smem_floats for L = 1, M = r
        return 4 * (255 * r + 2 * int(np.ceil(24 * r)) + 12)

    def accepted(r):
        return (255.0 * r + 2 * int(np.ceil(24 * r)) + 8) * 4 <= SMEM_BOUND

    below = max(r for r in range(2, 400) if launch_bytes(r) <= SMEM_OPT_IN)
    largest = max(r for r in range(2, 400) if accepted(r))
    assert (below, largest) == (40, 168)
    for r in (below, below + 1, largest):
        x = noise(1, 16000 * r // 2, seed=r)[0]
        check_sinc(oracle, conv().resample(x, 16000 * r), x, 16000 * r, 16000, ("ratio", r))
        oracle.sinc_design(16000 * r, 16000)
    # the next ratio; a rate off the grid; 4294967.297 Hz reduces to L = 4 294 967 297 >= 2^32
    for rin, rout, n in ((16000 * (largest + 1), 16000, 100000), (44100.0004, 16000, 100000), (16000, 4294967.297, 100)):
        with pytest.raises(ValueError):
            oracle.sinc_design(rin, rout)
        with pytest.raises(_lib.FluidAudioError) as e:
            conv(rout).resample(np.zeros(n, np.float32), rin)
        assert e.value.status == 8, (rin, rout, str(e.value))


def test_sinc_lengths_channels_and_layouts(gpu_lib, oracle):
    """Input lengths 0, 1, 2, H-1, H, 2H, 2H+1; output counts 0 and = 0, 1, 255 (mod 256); forced sinc on 3, 7 and 64
    channels in both layouts; int16 extremes."""
    for rin in (44100, 48000, 16001, 44100.001, 8000):
        d = oracle.sinc_design(rin, 16000)
        lengths = {0, 1, 2, d.half - 1, d.half, 2 * d.half, 2 * d.half + 1}
        lengths |= {frames_for(c, rin, 16000) for c in (256, 257, 511, 1024, 1025, 1279)} - {None}
        assert len(lengths) >= 10 or rin == 8000
        for n in sorted(lengths):
            x = noise(1, n, seed=n)[0]
            got = conv().resample_buffer(x[None], rin)
            assert got.size == oracle.resample_output_count(n, rin, 16000), (rin, n)
            check_sinc(oracle, got, x, rin, 16000, ("length", rin, n))
    assert oracle.resample_output_count(2, 44100, 16000) == 0    # inputs with no output at all are in the sweep
    sinc = conv(16000, Algorithm.sinc)
    for ch in (3, 7, 64):
        x = noise(ch, 9000, seed=ch)
        i16 = np.round(x * 32767).astype(np.int16)
        i16[:, 100] = -32768
        i16[:, 101] = 32767
        for pcm in (x, i16):
            got = sinc.resample_buffer(pcm, 44100)
            check_sinc(oracle, got, oracle.mixdown(pcm), 44100, 16000, ("forced sinc", ch, pcm.dtype))
            same_bits(sinc.resample_buffer(np.ascontiguousarray(pcm.T), 44100, interleaved=True), got, ("layout", ch))


# ------------------------------------------------------------------------------------------------ linear, bit for bit
def test_linear_bit_exact(gpu_lib, oracle):
    """AudioConverter.linearResample over every rate (fractional too), channels 3 to 64 (auto) and 1, 2 (forced), both
    layouts, float32 with NaN / Inf samples and int16 extremes."""
    lin = conv(16000, Algorithm.linear)
    rates = INT_RATES + FRACTIONAL
    for k, rin in enumerate(rates):
        for ch in (1, 2, 3 + k % 62):
            x = noise(ch, int(rin * 0.05) + k, seed=k * 7 + ch)
            if k % 3 == 0:
                x[ch - 1, x.shape[1] // 2] = (np.nan, np.inf, -np.inf)[k % 9 // 3]
            c = lin if ch <= 2 else conv()
            ref = oracle.linear_resample(x, rin, 16000) if rin != 16000 else oracle.mixdown(x)
            same_bits(c.resample_buffer(x, rin), ref, ("linear", rin, ch))
            same_bits(c.resample_buffer(np.ascontiguousarray(x.T), rin, interleaved=True), ref, ("linear il", rin, ch))
    for ch in range(3, 65):
        x = noise(ch, 1200 + ch, seed=ch)
        i16 = np.round(x * 32767).astype(np.int16)
        i16[0, 7], i16[ch - 1, 8] = -32768, 32767
        widened = i16.astype(np.float32) * np.float32(1.0 / 32768.0)
        same_bits(conv().resample_buffer(i16, 44100), oracle.linear_resample(widened, 44100, 16000), ("linear int16", ch))
        same_bits(conv().resample_buffer(x, 22050.25), oracle.linear_resample(x, 22050.25, 16000), ("linear", ch))


# ------------------------------------------------------------------------------------------------ non-finite input
@pytest.mark.parametrize("rin", [48000, 44100, 22050, 16001, 44100.001, 16000])
def test_non_finite_footprint(gpu_lib, oracle, rin):
    """A NaN / +Inf / -Inf at input m (start, middle, end, and the first and last input of a CTA's staged window): exactly
    the outputs whose 2H-tap window holds m are non-finite, every other output is bit-identical to the same call with that
    sample set to 0.  16 kHz stereo is the mixdown kernel: output m alone."""
    ch = 2 if rin == 16000 else 1
    n = int(rin * 0.2)
    x = noise(ch, n, seed=int(rin))
    count = oracle.resample_output_count(n, rin, 16000)
    if rin == 16000:
        positions = (0, 1, 255, 256, n // 2, n - 1)
    else:
        d = oracle.sinc_design(rin, 16000)
        n0, _ = oracle.sinc_positions(count, d.L, d.M)
        positions = (0, 1, n // 2, n - 1, int(n0[256]) - d.half + 1, int(n0[255]) + d.half, int(n0[512]) + d.half + 1,
                     int(n0[767]) + d.half + 2)
    for m in positions:
        base = x.copy()
        base[ch - 1, m] = 0.0
        ref = conv().resample_buffer(base, rin)
        want = np.zeros(count, bool)
        if rin == 16000:
            want[m] = True
        else:
            want = footprint(oracle, rin, 16000, count, m)
        assert want.any() or m >= n - 2, (rin, m)
        for v in (np.nan, np.inf, -np.inf):
            y = base.copy()
            y[ch - 1, m] = v
            got = conv().resample_buffer(y, rin)
            bad = ~np.isfinite(got)
            assert np.array_equal(bad, want), (rin, m, v, np.nonzero(bad != want)[0][:8])
            assert np.array_equal(got[~want].view(np.uint32), ref[~want].view(np.uint32)), (rin, m, v)


# ------------------------------------------------------------------------------------------------ invariants
def test_bitwise_invariants(gpu_lib, oracle):
    """int16 = the same values widened to float32 (v / 32768); interleaved = planar; forced sinc on C channels = sinc on
    the float32 mixdown as mono; an excerpt starting at s with s L / M whole reproduces the full call's interior outputs,
    with the CTA boundaries moved."""
    for rin, algo, ch in ((44100, Algorithm.auto, 2), (48000, Algorithm.auto, 1), (44100.001, Algorithm.auto, 2),
                          (16000, Algorithm.auto, 2), (22050, Algorithm.linear, 2), (44100, Algorithm.auto, 5)):
        c = conv(16000, algo)
        i16 = np.round(noise(ch, 7000, seed=ch) * 32767).astype(np.int16)
        i16[0, :2] = (-32768, 32767)
        wide = (i16.astype(np.float32) * np.float32(1.0 / 32768.0)).astype(np.float32)
        a = c.resample_buffer(i16, rin)
        same_bits(a, c.resample_buffer(wide, rin), ("int16 = widened", rin, ch))
        same_bits(a, c.resample_buffer(np.ascontiguousarray(i16.T), rin, interleaved=True), ("interleaved", rin, ch))
    sinc = conv(16000, Algorithm.sinc)
    for ch in (3, 7, 64):
        x = noise(ch, 5000, seed=ch)
        for rin in (44100, 16001):
            same_bits(sinc.resample_buffer(x, rin), conv().resample(oracle.mixdown(x), rin), ("sinc = mixdown", ch, rin))
    for rin, t in ((44100, 1), (44100, 3), (48000, 77), (16001, 1), (22050, 5)):
        d = oracle.sinc_design(rin, 16000)
        s, j = t * d.M, t * d.L                          # excerpt input s <-> full output j
        assert j % 256
        x = noise(1, s + 20000, seed=t)[0]
        full = conv().resample(x, rin)
        part = conv().resample(x[s:], rin)
        n0, _ = oracle.sinc_positions(part.size, d.L, d.M)
        inner = (n0 - d.half + 1 >= 0) & (n0 + d.half < x.size - s)
        assert inner.sum() > 1000
        same_bits(part[inner], full[j:j + part.size][inner], ("excerpt", rin, t))


# ------------------------------------------------------------------------------------------------ fused, multi-unit
def test_fused_pipeline_multi_unit(gpu_lib):
    """fa_audio_to_mel on inputs above 10 MB of PCM (several units: PCM copied and converted chunk by chunk) equals
    fa_mel_compute(fa_audio_resample(pcm)) bit for bit, for 1, 2, 7 and 24 pipeline units, both padding modes, both
    layouts."""
    t0 = time.time()
    rng = np.random.default_rng(11)
    cases = [
        ("48k stereo int16 interleaved, 10 min", 48000, (rng.integers(-32768, 32768, (48000 * 600, 2))).astype(np.int16),
         True),
        ("44.1k mono float32, 3 min", 44100, rng.uniform(-1, 1, 44100 * 180).astype(np.float32), False),
        ("48k 6-channel float32 (linear)", 48000, rng.uniform(-1, 1, (6, 48000 * 15)).astype(np.float32), False),
        ("44100.001 Hz mono float32", 44100.001, rng.uniform(-1, 1, 44100 * 80).astype(np.float32), False),
    ]
    m = AudioMelSpectrogram(n_mels=80)
    for what, rin, pcm, inter in cases:
        assert pcm.nbytes > 10 << 20, what
        mono = conv().resample_buffer(pcm, rin, interleaved=inter)
        for mode in (PaddingMode.center, PaddingMode.pre_padded):
            ref, rml, rnf = m.compute_flat_transposed(mono, last_audio_sample=0.2, padding_mode=mode)
            ref = ref.copy()
            for chunks in (1, 2, 7, 24):
                _lib.check(m._L.fa_mel_set_pipeline_chunks(m._h, chunks), "chunks")
                got, ml, nf, rs = m.compute_from_pcm(pcm, rin, interleaved=inter, last_audio_sample=0.2,
                                                     padding_mode=mode)
                assert (ml, nf, rs) == (rml, rnf, mono.size), (what, mode, chunks)
                same_bits(got, ref, (what, mode, chunks, "time-major"))
                got, _, _, _ = m.compute_from_pcm(pcm, rin, interleaved=inter, last_audio_sample=0.2, padding_mode=mode,
                                                  time_major=False)
                same_bits(got.reshape(80, nf).T, ref.reshape(nf, 80), (what, mode, chunks, "mel-major"))
    _lib.check(m._L.fa_mel_set_pipeline_chunks(m._h, 24), "chunks")
    print(f"fused multi-unit cases: {time.time() - t0:.1f} s")
