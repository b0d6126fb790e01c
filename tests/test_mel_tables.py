"""CPU tests of the log-mel plan's host tables (``fluidaudio_b200/csrc/mel_tables.cpp``), compiled with g++ behind a small C
shim (``tests/emul/mel_tables_shim.cpp``):

* the window and filterbank of every kind equal the oracle's bit for bit across nFFT 32..4096, 1..512 mels (counts with
  empty filters included), 8..48 kHz, both window kinds, Cohere's f_min / f_max and StyleTTS2's filter rate;
* the packed filterbank in both orders (swizzled for mel512_kernel, natural for mel_generic_kernel): every dense weight
  at its position with its scale, quad-aligned bands at their prefix-sum offsets, and mel512_kernel's schedule;
* the window placements and every rejection of the ex config check.
"""
import ctypes as C
import itertools

import numpy as np
import pytest

from mel_ex_restated import mel_tables_lib
from oracle import oracle_torch as OT

FB_AUDIO_MEL, FB_COHERE, FB_STYLETTS2, FB_LUXTTS = 0, 1, 2, 3   # FA_MEL_FB_*
EDGE_ZERO, EDGE_REFLECT = 0, 1                                  # FA_MEL_EDGE_*
NFFTS = [32, 64, 128, 256, 512, 1024, 2048, 4096]
RATES = [8000, 16000, 22050, 24000, 44100, 48000]
MELS = [1, 2, 3, 5, 23, 40, 64, 80, 100, 128, 200, 257, 400, 512]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return mel_tables_lib(str(tmp_path_factory.mktemp("mel_tables")))


def tables(L, sr, n_mels, n_fft, win, periodic, kind, filter_sr=0, f_min=0.0, f_max=0.0):
    w = np.zeros(win, np.float32)
    fb = np.zeros((n_mels, n_fft // 2 + 1), np.float32)
    L.mt_tables(sr, n_mels, n_fft, win, int(periodic), kind, filter_sr, f_min, f_max, w, fb.reshape(-1))
    return w, fb


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def grid():
    """(kind, sr, n_fft, n_mels, win, periodic, filter_sr, f_min, f_max): every kind x nFFT x rate, the mel counts, window
    lengths and kinds, Cohere bands and StyleTTS2 filter rates dealt round-robin."""
    mels = itertools.cycle(MELS)
    variant = itertools.count()
    for kind, n_fft, sr in itertools.product(range(4), NFFTS, RATES):
        for _ in range(2):
            v = next(variant)
            win = [n_fft, n_fft // 2 + 1, max(1, n_fft * 3 // 4), 2][v % 4]
            periodic = v % 3 == 0
            if win == 1 and not periodic and kind != FB_COHERE:
                win = 2   # a symmetric window of one sample divides by zero in every class but Cohere's
            filter_sr, f_min, f_max = 0, 0.0, 0.0
            if kind == FB_COHERE:
                f_min, f_max = [(0.0, 0.0), (0.0, sr / 2), (20.0, 0.0), (125.0, 0.3 * sr)][v % 4]
                if v % 5 == 0:
                    win = 1
            elif kind == FB_STYLETTS2:
                filter_sr = [0, 16000, 8000][v % 3]
            yield kind, sr, n_fft, next(mels), win, periodic, filter_sr, f_min, f_max


def oracle_tables(oracle, kind, sr, n_fft, n_mels, win, periodic, filter_sr, f_min, f_max):
    fr = filter_sr or sr
    if kind == FB_COHERE and not periodic:
        w = OT.cohere_window(win)
    elif kind == FB_STYLETTS2 and periodic:
        off = (n_fft - win) // 2
        w = OT.styletts2_window(win, n_fft)[off:off + win]
    elif kind == FB_LUXTTS and periodic:
        w = OT.luxtts_window(win)
    else:
        w = oracle.hann_window(win, periodic)
    if kind == FB_AUDIO_MEL:
        fb = oracle.mel_filterbank(n_fft, n_mels, fr)
    elif kind == FB_COHERE:
        fb = OT.cohere_filterbank(fr, n_fft, n_mels, f_min, f_max if f_max > 0 else fr / 2)
    elif kind == FB_STYLETTS2:
        fb = OT.styletts2_filterbank(n_mels, n_fft, fr)
    else:
        fb = OT.luxtts_filterbank(n_fft, n_mels, fr)
    return w, fb


def test_tables_of_every_kind_are_bit_identical_to_the_oracle(lib, oracle):
    seen_empty = 0
    for cfg in grid():
        kind, sr, n_fft, n_mels, win, periodic, filter_sr, f_min, f_max = cfg
        w, fb = tables(lib, sr, n_mels, n_fft, win, periodic, kind, filter_sr, f_min, f_max)
        ow, ofb = oracle_tables(oracle, *cfg)
        assert same_bits(w, ow), cfg
        assert same_bits(fb, ofb), cfg
        seen_empty += int((~fb.any(axis=1)).any())
    assert seen_empty > 10   # the grid reaches mel counts whose narrow filters catch no bin


def pow_pos(k):
    return k ^ ((k >> 4) & 3)


def pack(L, fb, swizzled, scale):
    n_mels, bins = fb.shape
    fb = np.ascontiguousarray(fb, np.float32).reshape(-1)
    nnz, n_slots = C.c_int32(), C.c_int32()
    L.mt_pack_sizes(fb, n_mels, bins, C.byref(nnz), C.byref(n_slots))
    lo, hi, off = (np.zeros(n_mels, np.int32) for _ in range(3))
    w = np.zeros(max(nnz.value, 1), np.float32)
    slots = np.zeros((max(n_slots.value, 1), 4), np.int32)
    L.mt_pack(fb, n_mels, bins, int(swizzled), scale, lo, hi, off, w, slots.reshape(-1))
    return lo, hi, off, w[:nnz.value], slots[:n_slots.value]


def check_packing(L, fb, swizzled, scale, warps):
    n_mels, bins = fb.shape
    lo, hi, off, w, slots = pack(L, fb, swizzled, scale)
    # bands: the non-zero bins widened to whole quads, weights at the prefix sums of the band widths
    for m in range(n_mels):
        nz = np.flatnonzero(fb[m])
        want = (int(nz[0]) & ~3, (int(nz[-1]) + 4) & ~3) if nz.size else (0, 0)
        assert (lo[m], hi[m]) == want, m
    assert (lo % 4 == 0).all() and (hi % 4 == 0).all() and (hi >= lo).all()
    assert off.tolist() == np.concatenate([[0], np.cumsum(hi - lo)[:-1]]).tolist() and w.size == int((hi - lo).sum())
    # weights: position k of a band holds bin pow_pos(k) (k in natural order) times scale, zero past the last bin
    want = np.zeros_like(w)
    placed = np.zeros(fb.shape, np.int32)
    for m in range(n_mels):
        for k in range(lo[m], hi[m]):
            src = pow_pos(k) if swizzled else k
            assert src >> 2 == k >> 2   # a permutation inside the bin quad
            if src < bins:
                want[off[m] + k - lo[m]] = np.float32(scale) * fb[m, src]
                placed[m, src] += 1
    assert same_bits(w, want)
    assert (placed[fb != 0] == 1).all()   # every non-zero dense weight exactly once, every other packed weight zero
    assert np.count_nonzero(w) == np.count_nonzero(fb)
    # schedule: slot (iteration * warps + warp) * 4 + member; a (iteration, warp) holds the four mels of one group
    assert slots.shape[0] % (4 * warps) == 0
    mels = []
    for s0 in range(0, slots.shape[0], 4):
        group = slots[s0:s0 + 4]
        if (group[:, 3] < 0).all():
            assert (group == [0, 0, 0, -1]).all()
            continue
        g = group[0, 3] // 4
        assert group[0, 3] == 4 * g
        for q in range(4):
            m = 4 * g + q
            if m < n_mels:
                assert group[q].tolist() == [lo[m], (hi[m] - lo[m]) >> 2, off[m], m]
                mels.append(m)
            else:
                assert group[q].tolist() == [0, 0, 0, -1]
    assert sorted(mels) == list(range(n_mels))


def test_packed_filterbank_in_both_orders(lib):
    warps = lib.mt_warps_per_cta()
    assert warps == 8
    for i, cfg in enumerate(grid()):
        if i % 3:
            continue
        kind, sr, n_fft, n_mels, win, periodic, filter_sr, f_min, f_max = cfg
        _, fb = tables(lib, sr, n_mels, n_fft, win, periodic, kind, filter_sr, f_min, f_max)
        swizzled = n_fft == 512 and i % 2 == 0
        check_packing(lib, fb, swizzled, 0.25 if i % 4 == 0 else 1.0, warps)
    # the specialised kernel's tables at the shapes its callers use, both orders
    for n_mels, sr in ((80, 16000), (128, 16000), (1, 8000), (5, 48000), (512, 16000), (200, 8000)):
        _, fb = tables(lib, sr, n_mels, 512, 400, False, FB_AUDIO_MEL)
        for swizzled in (True, False):
            check_packing(lib, fb, swizzled, 0.25, warps)


def test_window_placements(lib):
    for n_fft, win in ((512, 400), (512, 512), (256, 200), (32, 1), (4096, 2049)):
        w = (np.arange(win, dtype=np.float32) + 1) / win
        for off in ((n_fft - win) // 2, 0):
            wt, it = np.full(n_fft, 7, np.float32), np.full(n_fft, 7, np.uint8)
            lib.mt_place_window(w, win, n_fft, off, wt, it)
            want = np.zeros(n_fft, np.float32)
            want[off:off + win] = w
            assert same_bits(wt, want) and it.tolist() == (want != 0).astype(np.uint8).tolist()


def test_ex_config_check(lib):
    def check(kind=FB_AUDIO_MEL, filter_sr=0, f_min=0.0, f_max=0.0, edge=EDGE_ZERO, preemph=0.97, power=2.0, mean=0.0,
              std=1.0, sr=16000):
        r = lib.mt_check(sr, kind, filter_sr, f_min, f_max, edge, preemph, power, mean, std)
        return r.decode() if r is not None else None

    nan, inf = float("nan"), float("inf")
    assert check() is None                                                            # fa_mel_create's config
    assert check(FB_COHERE, f_max=8000.0) is None                                     # the presets
    assert check(FB_STYLETTS2, filter_sr=16000, edge=EDGE_REFLECT, preemph=0.0, mean=-4.0, std=4.0, sr=24000) is None
    assert check(FB_LUXTTS, edge=EDGE_REFLECT, preemph=0.0, power=1.0, sr=24000) is None
    assert check(f_max=8000.0) is None and check(FB_STYLETTS2, filter_sr=16000, f_max=8000.0) is None
    assert check(FB_COHERE, f_min=300.0, f_max=3000.0, power=1.5) is None
    for kind in (-1, 4):
        assert "filterbank must be one of FA_MEL_FB_*" in check(kind)
    assert "filter_sample_rate must be 0" in check(filter_sr=-1)
    for edge in (-1, 2):
        assert "center_edge must be" in check(edge=edge)
    for power in (0.0, -1.0, nan, inf):
        assert "spectrum_power must be finite" in check(power=power)
    for mean, std in ((nan, 1.0), (inf, 1.0), (0.0, 0.0), (0.0, nan), (0.0, -inf)):
        assert "log_mean must be finite" in check(mean=mean, std=std)
    for f_min, f_max in ((nan, 0.0), (0.0, inf), (-inf, 8000.0)):
        assert "f_min and f_max must be finite" in check(FB_COHERE, f_min=f_min, f_max=f_max)
    for kind in (FB_AUDIO_MEL, FB_STYLETTS2, FB_LUXTTS):
        assert "apply to FA_MEL_FB_COHERE only" in check(kind, f_min=10.0, preemph=0.0)
        assert "apply to FA_MEL_FB_COHERE only" in check(kind, f_max=7000.0, preemph=0.0)
    assert "apply to FA_MEL_FB_COHERE only" in check(FB_STYLETTS2, filter_sr=16000, f_max=12000.0, sr=24000)
    assert "FA_MEL_EDGE_REFLECT needs preemph 0" in check(edge=EDGE_REFLECT)
