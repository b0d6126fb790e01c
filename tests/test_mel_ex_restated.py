"""CPU checks of the float64 restatement of an ex handle's log-mel and of its derived bar (tests/mel_ex_restated.py).

* The restatement agrees with the per-class float64 restatements written from the Swift (``np_cohere``,
  ``np_styletts2``, ``np_luxtts`` in test_mel_torch_frontends.py) to 1e-9, on the presets and on every class parameter
  those functions take.
* The float32 oracles lie within the bar of the restatement: ``oracle_torch``'s three classes at the same variations
  (Cohere's log-mel before its CMVN, on clips of one valid frame; its two-rounded pre-emphasis adds u |a x[i-1]| per
  sample to S_f) and ``oracle.py``'s AudioMelSpectrogram log-mel for neutral handles in all three modes.
* The bar has teeth: each restated defect (MUTATIONS) exceeds the bar on at least one case of the GPU sweep's
  configurations and inputs, with the tables the handles build (``mt_tables``).
"""
import numpy as np
import pytest

import mel_ex_restated as R
from mel_ex_restated import CENTER, LEGACY, PRE_PADDED, Cfg
from oracle import oracle_torch as OT
from test_mel_torch_frontends import _hann, np_cohere, np_cohere_filterbank, np_htk_filterbank, np_luxtts, np_styletts2

F32 = np.float32


@pytest.fixture(scope="module")
def tables(tmp_path_factory):
    L = R.mel_tables_lib(str(tmp_path_factory.mktemp("mel_ex")))
    return lambda cfg: R.cpu_tables(L, cfg)


@pytest.fixture(scope="module")
def packer(tmp_path_factory):
    return R.mel_tables_lib(str(tmp_path_factory.mktemp("mel_pack")))


def _audio(n, rate=16000, seed=1):
    rng = np.random.default_rng(seed + n)
    return (R.signal("speech", n, rate) + 0.05 * rng.standard_normal(n)).astype(F32)


def f32(v):
    """A constant as the handle holds it (the class restatements take float64 constants)."""
    return float(F32(v))


def _close(got, ref, what):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    d = np.abs(got - ref)
    assert (d <= 1e-9 * (1.0 + np.abs(ref))).all(), (what, float((d / (1.0 + np.abs(ref))).max()))


def _placed(window, n_fft):
    w = np.zeros(n_fft)
    w[(n_fft - window.size) // 2:(n_fft - window.size) // 2 + window.size] = window
    return w


def _cmvn64(L, valid):
    """np_cohere's CMVN and zeroing on a [T x M] log-mel -> [M x T]."""
    mel = L.T.copy()
    if valid > 1:
        v = mel[:, :valid]
        sd = np.sqrt(((v - v.mean(1, keepdims=True)) ** 2).sum(1, keepdims=True) / (valid - 1))
        mel[:, :valid] = (v - v.mean(1, keepdims=True)) / (sd + 1e-5)
    mel[:, valid:] = 0.0
    return mel


COHERE_VARIANTS = [dict(), dict(power=1.0), dict(power=1.5), dict(win=401), dict(win=1000), dict(hop=161),
                   dict(hop=441), dict(n_mels=1), dict(n_mels=64), dict(n_mels=257), dict(f_min=125.0, f_max=3000.0),
                   dict(f_min=20.0, f_max=0.0), dict(preemph=0.0), dict(sr=22050, f_max=11025.0)]
STYLETTS2_VARIANTS = [dict(), dict(n_fft=1024, win=1024), dict(n_fft=4096, win=2401), dict(win=1201), dict(hop=301),
                      dict(hop=2500), dict(n_mels=1), dict(n_mels=257), dict(filter_sr=22050), dict(filter_sr=24000),
                      dict(mean=1.5, std=-0.37)]
LUXTTS_VARIANTS = [dict(), dict(n_fft=512), dict(n_fft=2048), dict(hop=255), dict(n_mels=1), dict(n_mels=257),
                   dict(sr=16000), dict(sr=48000), dict(floor=1e-5), dict(floor=1e-10)]


def cohere_cfg(sr=16000, win=400, hop=160, n_mels=128, f_min=0.0, f_max=8000.0, preemph=0.97, power=2.0):
    n_fft = 1 << max(0, (win - 1).bit_length())
    return Cfg(sample_rate=sr, n_mels=n_mels, n_fft=n_fft, hop=hop, win=win, preemph=preemph, floor=2.0 ** -24,
               kind=R.FB_COHERE, f_min=f_min, f_max=f_max, power=power)


def styletts2_cfg(n_fft=2048, win=1200, hop=300, n_mels=80, filter_sr=16000, mean=-4.0, std=4.0):
    return Cfg(sample_rate=24000, n_mels=n_mels, n_fft=n_fft, hop=hop, win=win, preemph=0.0, floor=1e-5, periodic=True,
               kind=R.FB_STYLETTS2, filter_sr=filter_sr, reflect=True, mean=mean, std=std)


def luxtts_cfg(n_fft=1024, hop=256, n_mels=100, sr=24000, floor=1e-7):
    return Cfg(sample_rate=sr, n_mels=n_mels, n_fft=n_fft, hop=hop, win=n_fft, preemph=0.0, floor=floor, clamped=True,
               periodic=True, kind=R.FB_LUXTTS, reflect=True, power=1.0)


# ================================================================================================ pinned to the classes
@pytest.mark.parametrize("v", COHERE_VARIANTS, ids=str)
def test_restatement_equals_np_cohere(v):
    c = cohere_cfg(**v)
    for n in (0, 1, 2, c.n_fft // 2, c.hop + 3, 2 * c.hop + 1, 16000 + 7):
        a = _audio(n)
        T, valid = 1 + n // c.hop, n // c.hop
        w = _placed(_hann(c.win, False), c.n_fft)[(c.n_fft - c.win) // 2:][:c.win]
        fb = np_cohere_filterbank(c.sample_rate, c.n_fft, c.n_mels, c.f_min, c.f_max or c.sample_rate / 2)
        r = R.restate(c, w, fb, a, CENTER, 0.0, T)
        ref, rvalid = np_cohere(a, c.sample_rate, c.win, c.hop, c.n_mels, c.f_min, c.f_max or c.sample_rate / 2,
                                f32(c.preemph), c.power, f32(c.floor))
        assert rvalid == valid
        _close(_cmvn64(r.out, valid), ref, (v, n))


@pytest.mark.parametrize("v", STYLETTS2_VARIANTS, ids=str)
def test_restatement_equals_np_styletts2(v):
    c = styletts2_cfg(**v)
    for n in (0, 1, 2, 5, c.n_fft // 2 - 1, c.n_fft // 2, c.n_fft // 2 + 1, 3 * c.hop + 1, 24000 + 5):
        a = _audio(n, 24000)
        T = 1 + n // c.hop
        r = R.restate(c, _hann(c.win, True), np_htk_filterbank(c.n_fft, c.n_mels, c.filter_sr), a, CENTER, 0.0, T)
        ref = np_styletts2(a, c.n_fft, c.win, c.hop, c.n_mels, c.filter_sr, f32(c.mean), f32(c.std), f32(c.floor))
        _close(r.out.T, ref, (v, n))


@pytest.mark.parametrize("v", LUXTTS_VARIANTS, ids=str)
def test_restatement_equals_np_luxtts(v):
    c = luxtts_cfg(**v)
    for n in (1, 2, c.hop // 2, c.n_fft // 2, c.n_fft // 2 + 1, 3 * c.hop + 1, 24000 + 5):
        a = _audio(n, c.sample_rate)
        T = (n + c.hop // 2) // c.hop
        r = R.restate(c, _hann(c.n_fft, True), np_htk_filterbank(c.n_fft, c.n_mels, c.sample_rate), a, CENTER, 0.0, T)
        _close(r.out, np_luxtts(a, c.n_fft, c.hop, c.n_mels, c.sample_rate, f32(c.floor)), (v, n))


# ================================================================================================ the oracles in the bar
def _within(got, cfg, r, what, worst):
    worst[0] = max(worst[0], R.compare(got, cfg, r, what))


def test_oracles_lie_within_the_bar(oracle, tables):
    worst = {k: [0.0] for k in ("cohere", "styletts2", "luxtts", "audio_mel")}
    for v in COHERE_VARIANTS:
        c = cohere_cfg(**v)
        w, fb = tables(c)
        kw = dict(sample_rate=c.sample_rate, win_length=c.win, hop_length=c.hop, n_mels=c.n_mels, f_min=c.f_min,
                  f_max=c.f_max or c.sample_rate / 2, preemph=c.preemph, mag_power=c.power)
        for kind in ("noise", "speech", "tone"):
            for n in (c.hop, c.hop + c.hop // 2, 2 * c.hop - 1):   # one valid frame: the log-mel before CMVN
                a = R.signal(kind, n, c.sample_rate, seed=n)
                got, valid = OT.cohere_compute(a, **kw)
                assert valid == 1
                r = R.restate(c, w, fb, a, CENTER, 0.0, 1, preemph_two_roundings=True)
                _within(got[:, :1].T, c, r, ("cohere", v, kind, n), worst["cohere"])
    for v in STYLETTS2_VARIANTS:
        c = styletts2_cfg(**v)
        w, fb = tables(c)
        for kind in ("noise", "speech"):
            for n in (1, 2, c.n_fft // 2, c.n_fft // 2 + 1, 5 * c.hop + 1, 24000 + 11):
                a = R.signal(kind, n, 24000, seed=n)
                got, T = OT.styletts2_compute(a, n_fft=c.n_fft, win_length=c.win, hop_length=c.hop, n_mels=c.n_mels,
                                              filter_sample_rate=c.filter_sr, mean=c.mean, std=c.std)
                r = R.restate(c, w, fb, a, CENTER, 0.0, T)
                _within(got.T, c, r, ("styletts2", v, kind, n), worst["styletts2"])
    for v in LUXTTS_VARIANTS:
        c = luxtts_cfg(**v)
        w, fb = tables(c)
        for kind in ("noise", "speech"):
            for n in (1, 2, c.n_fft // 2, c.n_fft // 2 + 1, 5 * c.hop + 1, 24000 + 11):
                a = R.signal(kind, n, c.sample_rate, seed=n)
                got = OT.luxtts_extract(a, n_fft=c.n_fft, hop_length=c.hop, n_mels=c.n_mels, sample_rate=c.sample_rate,
                                        log_floor=c.floor)
                r = R.restate(c, w, fb, a, CENTER, 0.0, got.shape[0])
                _within(got, c, r, ("luxtts", v, kind, n), worst["luxtts"])
    for n_fft, win, hop, n_mels, sr, preemph, clamped, periodic in (
            (512, 400, 160, 128, 16000, 0.97, False, False), (256, 200, 80, 23, 8000, 0.0, True, True),
            (1024, 1024, 161, 80, 48000, 0.97, False, False), (64, 33, 7, 3, 16000, 0.5, True, False)):
        c = Cfg(sample_rate=sr, n_mels=n_mels, n_fft=n_fft, hop=hop, win=win, preemph=preemph,
                floor=1e-10 if clamped else 2.0 ** -24, clamped=clamped, periodic=periodic)
        w, fb = tables(c)
        ocfg = oracle.mel_config(sr, n_mels, n_fft, hop, win, preemph, 0, c.floor, int(clamped), periodic)
        for mode in (CENTER, PRE_PADDED, LEGACY):
            for n in (n_fft + 3 * hop + 1, 8000 + 13):
                a = R.signal("speech", n, sr, seed=n)
                if mode == LEGACY:
                    mel, T = oracle.mel_legacy(ocfg, a)
                    got = np.asarray(mel, np.float64).reshape(n_mels, -1).T[:T]
                else:
                    got, T, _ = oracle.mel_flat_transposed(ocfg, a, 0.125, mode)
                    got = got[:T]
                r = R.restate(c, w, fb, a, mode, 0.125 if mode != LEGACY else 0.0, T)
                _within(got, c, r, ("audio_mel", n_fft, mode, n), worst["audio_mel"])
    print("\noracles, worst |d| / bar: " + ", ".join(f"{k} {v[0]:.3g}" for k, v in worst.items()))


# ================================================================================================ the bar has teeth
def _exceeds(cfg, w, fb, a, mode, mutation):
    r = R.restate(cfg, w, fb, a, mode)
    m = R.restate(cfg, w, fb, a, mode, mutate=mutation)
    b, _ = R.bar(cfg, r)
    fin = np.isfinite(r.out) & np.isfinite(m.out) & np.isfinite(b)
    return bool((np.abs(m.out - r.out)[fin] > b[fin]).any())


def _applies(cfg, n, mutation):
    if mutation in ("torch_reflect", "preemph_reflect"):
        return cfg.reflect and (mutation != "torch_reflect" or 2 <= n <= cfg.n_fft // 2)
    if mutation == "power2":
        return cfg.power == 1.5
    if mutation == "affine_order":
        return cfg.affine
    return True


@pytest.mark.parametrize("mutation", R.MUTATIONS)
def test_each_restated_defect_exceeds_the_bar(tables, mutation):
    tried = 0
    for cfg in R.sweep_configs():
        if cfg.n_fft > 2048 or cfg.hop == 1:
            continue   # the sweep's other configurations cover every mutation; these only cost time here
        w, fb = tables(cfg)
        for n in R.clip_lengths(cfg, cfg.sample_rate):
            if n == 0 or not _applies(cfg, n, mutation):
                continue
            for kind in ("noise", "speech", "square", "dc", "tone"):
                tried += 1
                a = R.signal(kind, n, cfg.sample_rate, seed=n)
                if _exceeds(cfg, w, fb, a, CENTER, mutation):
                    print(f"\n{mutation}: exceeds the bar at {cfg}, n {n}, {kind} (after {tried} cases)")
                    return
    pytest.fail(f"{mutation} stays inside the bar on all {tried} cases")


def test_sweep_reaches_every_variant_and_axis():
    cfgs = R.sweep_configs()
    hist = {v: 0 for v in R.VARIANTS}
    for c in cfgs:
        hist[c.variant(CENTER)] += 1
        assert c.generic()
    assert min(hist.values()) >= 3, hist
    assert {c.n_fft for c in cfgs} == set(R.NFFTS) and {c.kind for c in cfgs} == {0, 1, 2, 3}
    assert {c.n_mels for c in cfgs} == set(R.MELS) and {c.power for c in cfgs} >= {0.5, 1.5, 3.0, 1.0, 2.0}
    wins = {(c.win == c.n_fft, c.win == c.n_fft - 1, c.win == c.n_fft // 2 + 1, c.win == 1) for c in cfgs}
    assert len(wins) == 4
    assert any(c.hop == 1 for c in cfgs) and any(c.hop > c.n_fft for c in cfgs) and any(c.hop == c.win for c in cfgs)
    assert {(c.clamped, c.floor) for c in cfgs} == set(R.FLOORS)


def test_restated_bands_are_the_packers(tables, packer):
    """The bar's band widths (nq) are those of pack_bands, on every table of the sweep and of the class variations."""
    cfgs = R.sweep_configs() + [cohere_cfg(**v) for v in COHERE_VARIANTS] + [styletts2_cfg(**v) for v in STYLETTS2_VARIANTS]
    cfgs += [luxtts_cfg(**v) for v in LUXTTS_VARIANTS]
    for cfg in cfgs:
        _, fb = tables(cfg)
        lo, hi = R.bands(fb)
        plo, phi = R.packed_bands(packer, fb)
        assert np.array_equal(lo, plo) and np.array_equal(hi, phi), cfg


def test_bar_covers_subnormal_intermediates():
    """With a log floor of 0, mel values in the subnormal range: the bar's absolute terms keep it above the float32
    roundings there (|X|^3, the weight products and the sum emulated in float32).  Without them this case exceeds the
    relative bar more than a hundredfold."""
    cfg = Cfg(n_mels=3, n_fft=64, hop=16, win=64, preemph=0.0, floor=0.0, clamped=False, power=3.0, periodic=True)
    w = np.hanning(64).astype(F32)
    fb = np.zeros((3, 33), F32)
    fb[:, 4:12] = 0.5
    a = (np.random.default_rng(2).standard_normal(200) * 1e-15).astype(F32)   # mel values ~1e-42
    r = R.restate(cfg, w, fb, a, CENTER)
    assert ((r.E > 0) & (r.E < 2.0 ** -126)).any()
    b, _ = R.bar(cfg, r)
    E32 = np.zeros_like(r.E)
    spec = (r.absX.astype(F32) ** F32(3)).astype(F32)
    for m in range(3):
        acc = np.zeros(r.E.shape[0], F32)
        for k in range(4, 12):
            acc = (acc + F32(0.5) * spec[:, k]).astype(F32)
        E32[:, m] = acc
    with np.errstate(divide="ignore"):
        L32 = np.log(E32.astype(np.float64))
    fin = np.isfinite(L32) & np.isfinite(r.out)
    assert fin.any() and (np.abs(L32[fin] - r.out[fin]) <= b[fin]).all()
