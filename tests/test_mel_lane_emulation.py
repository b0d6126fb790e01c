"""The host emulation of mel512_kernel's log argument (tests/mel_lane_emulated.py, tests/emul/mel_lane_emul.cpp) on the
CPU: its filterbank stage against float64 and against the older emulator's ``mel_dot``, its whole path against
``mel_emul`` / ``mel_emul_f32x2``, and the defects it exists to catch.  tests/test_gpu_mel_emulated.py holds the kernel to
it on the GPU.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import mel_lane_emulated as ME
from fluidaudio_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U, TINY, F32 = ME.U, ME.TINY, ME.F32


def dot_bar(E, nq):
    """(4 nq + 1) u E: a chain of 4 nq fmaf over non-negative terms (plus absolute rounding where E is subnormal)."""
    return (4 * nq + 1) * (U * np.abs(E) + TINY)


def power_rows(rng, rows):
    """Power rows 4|X|^2 spanning normal, tiny and subnormal magnitudes, with exact zeros."""
    p = rng.exponential(1.0, (rows, ME.BINS)) * 10.0 ** rng.uniform(-8, 8, (rows, 1))
    p[rows // 4: rows // 2] *= 1e-38                    # subnormal rows
    p[:, rng.integers(0, ME.BINS, 9)] = 0.0
    return p.astype(F32)


@pytest.mark.parametrize("nm,sr", [(1, 16000), (23, 8000), (80, 16000), (128, 22050), (257, 48000), (512, 16000)])
def test_device_order_band_sum_within_the_dot_bar(oracle, nm, sr):
    """E in the device's order (quad-rounded band, swizzled positions, one fmaf chain) equals the float64 band sum of the
    same power row within (4 nq + 1) u E, and the host-order mel_dot (separate multiply and add) within the same bar."""
    fb = oracle.mel_filterbank(512, nm, sr)
    lo, hi = ME.quad_bands(fb)
    nq = (hi - lo) // 4
    p = power_rows(np.random.default_rng(nm), 64)
    E, _ = ME.lane_dot(p, fb)
    Ed, _ = ME.lane_dot(p, fb, defects=ME.DEFECTS["dot_mul_add"])
    w = (F32(0.25) * fb).astype(np.float64)
    E64 = p.astype(np.float64) @ w.T
    assert (np.abs(E - E64) <= dot_bar(E64, nq)).all()
    assert (np.abs(Ed - E64) <= dot_bar(E64, nq)).all()
    assert (np.abs(E - Ed) <= dot_bar(np.maximum(E, Ed), nq)).all()
    assert not np.array_equal(E, Ed), "the two orders never differ: the comparison is vacuous"
    empty = ~fb.any(axis=1)
    assert (E[:, empty] == 0).all()


@pytest.mark.parametrize("bad", [np.inf, np.nan])
def test_non_finite_bin_inside_the_quad_range_poisons_the_mel(oracle, bad):
    """A NaN or inf bin inside a mel's quad-rounded range but outside its filter's band makes the mel NaN (the zero weight
    times inf is NaN, as on the device), in both floor modes at every log floor; the bare-band mel_dot stays finite."""
    fb = oracle.mel_filterbank(512, 80)
    lo, hi = ME.quad_bands(fb)
    seen = 0
    for m in range(fb.shape[0]):
        nz = np.flatnonzero(fb[m])
        outside = [k for k in range(lo[m], min(hi[m], ME.BINS)) if fb[m, k] == 0 and (k < nz[0] or k > nz[-1])]
        if not outside:
            continue
        seen += 1
        p = power_rows(np.random.default_rng(m), 1)
        p[0, outside[0]] = bad
        for clamped in (0, 1):
            for fl in ME.FLOORS:
                E, x = ME.lane_dot(p, fb, fl, clamped)
                assert np.isnan(E[0, m]) and np.isnan(x[0, m]), (m, clamped, fl)
                Ed, _ = ME.lane_dot(p, fb, fl, clamped, defects=ME.DEFECTS["dot_mul_add"])
                assert np.isfinite(Ed[0, m]), m
                # every other mel whose quad range misses the bin is finite
                others = (lo > outside[0]) | (hi <= outside[0])
                assert np.isfinite(E[0, others]).all()
    assert seen >= 20, seen


def _mel_emul_lib(tmp_path):
    out = str(tmp_path / "libmel_emul.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "emul", "mel_emul.cpp")])
    L = C.CDLL(out)
    f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
    args = [f32p, C.c_longlong, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, f32p, f32p, C.c_float,
            C.c_int, C.c_longlong, f32p]
    L.mel_emul.argtypes = L.mel_emul_f32x2.argtypes = args
    return L


def test_end_to_end_matches_mel_emul(tmp_path, oracle):
    """On the CPU sweep's axes (tests/test_host_logic.py): the new entry's logs (host libm) equal mel_emul's /
    mel_emul_f32x2's bit for bit wherever the device order and the host order give the same E; elsewhere the two E agree
    within the dot bar.  The entry's mel_dot defect reproduces mel_emul everywhere, which pins the rest of the path."""
    L = _mel_emul_lib(tmp_path)
    hops = (2, 64, 128, 158, 256, 320, 512, 514, 1000)
    wins = (512, 449, 448, 400, 385, 384, 383, 256, 64)
    mels = (1, 3, 23, 40, 81, 128, 200, 257)
    rates = (8000, 22050, 48000, 16000)
    floors = (2.0 ** -24, 1e-10, 1e-38, 0.0)
    i = differ = 0
    for hop in hops:
        for win in wins:
            for mode in (0, 1, 2):
                nm, sr, fl = mels[i % len(mels)], rates[i % len(rates)], floors[i % len(floors)]
                clamped, pre = (i // len(floors)) % 2, (0.97 if (i // 2) % 2 == 0 else 0.0)
                i += 1
                off = 0 if mode == 2 else (512 - win) // 2
                pad = 256 if mode == 0 else 0
                pre = 0.0 if mode == 2 else pre
                frames = (17, 33, 2, 16, 1, 31, 15)[i % 7]
                x = synth.tone_noise_audio(max(1, (frames - 1) * hop + 512 - pad), seed=i)
                T = ME.frame_count(x.size, hop, win, mode)
                fb = oracle.mel_filterbank(512, nm, sr)
                w = oracle.hann_window(win)
                nq = np.diff(np.stack(ME.quad_bands(fb)), axis=0)[0] // 4
                for f32, fn in ((False, L.mel_emul), (True, L.mel_emul_f32x2)):
                    what = dict(hop=hop, win=win, mode=mode, n_mels=nm, sr=sr, floor=fl, clamped=clamped, f32=f32)
                    ref = np.zeros((T, nm), F32)
                    assert fn(x, x.size, 0.3, hop, win, off, pad, F32(pre), nm, fb, w, F32(fl), clamped, T, ref) == 0
                    _, E, _, out = ME.lane_frames(f32, x, 0.3, hop, w, off, pad, pre, fb, fl, clamped, T, libm_log=True)
                    _, Ed, _, outd = ME.lane_frames(f32, x, 0.3, hop, w, off, pad, pre, fb, fl, clamped, T,
                                                    defects=ME.DEFECTS["dot_mul_add"], libm_log=True)
                    assert np.array_equal(outd, ref, equal_nan=True), what
                    same = (E == Ed) | (np.isnan(E) & np.isnan(Ed))
                    assert np.array_equal(out[same], ref[same], equal_nan=True), what
                    assert (np.abs(E - Ed)[~same] <= dot_bar(np.maximum(E, Ed), np.broadcast_to(nq, E.shape))[~same]).all(), what
                    differ += int((~same).sum())
    assert i == len(hops) * len(wins) * 3
    assert differ > 0, "the two orders never differ on the sweep: the bar comparison is vacuous"


def _old_f32_bar(r, top):   # tests/test_gpu_mel_sweep.py's bar against the FP64 oracle
    with np.errstate(over="ignore"):
        return np.minimum(2e-3, 1e-4 * np.maximum(1.0, np.exp(top - r - 12.0)))


def _oracle_rows(oracle, cfg, x, last, mode, T):
    if mode == ME.LEGACY:
        ref, T2 = oracle.mel_legacy(cfg, x)
        return ref.T[:T]
    ref, ml, nf = oracle.mel_flat_transposed(cfg, x, last=last, padding_mode=mode)
    return ref.reshape(nf, cfg.n_mels)[:T]


def test_every_defect_exceeds_the_bar(oracle):
    """Each defect flag moves some log-mel entry of the GPU sweep's inputs (tests/test_gpu_mel_emulated.py) by more than
    twice the float32 bar: a kernel with that defect fails the GPU comparison whatever its log's own error.  The table also
    says which defects the oracle comparison's bar (1e-4 .. 2e-3) lets through.  The one exception changes no output at
    all (ME.INVISIBLE: the sample it moves is always multiplied by a zero window coefficient), which is asserted too."""
    worst = {k: 0.0 for k in ME.DEFECTS}
    old_caught = {k: False for k in ME.DEFECTS}
    for c in ME.cross_cases():
        n = ME.length_for(c["frames"], c["hop"], c["win"], c["mode"])
        x = ME.signal(c["signal"], n, c["seed"], c["sr"])
        T = ME.frame_count(n, c["hop"], c["win"], c["mode"])
        off, pad, pre = ME.placement(c, c["mode"])
        fb = oracle.mel_filterbank(512, c["n_mels"], c["sr"])
        w = oracle.hann_window(c["win"])
        args = (x, c["last"], c["hop"], w, off, pad, pre, fb, c["floor"], c["clamped"], T)
        _, _, x0, y0 = ME.lane_frames(True, *args, libm_log=True)
        cfg = oracle.mel_config(sample_rate=c["sr"], n_mels=c["n_mels"], hop_length=c["hop"], win_length=c["win"],
                                preemph=c["preemph"], log_floor=c["floor"], log_floor_mode=c["clamped"])
        ref = _oracle_rows(oracle, cfg, x, c["last"], c["mode"], T)
        fin_r = np.isfinite(ref)
        top = np.broadcast_to(np.where(fin_r, ref, -np.inf).max(axis=1, keepdims=True), ref.shape)

        def old_fails(y):
            """Entries the oracle comparison rejects (outside its bar, or finite where the oracle is not or vice versa)."""
            with np.errstate(invalid="ignore"):
                return np.where(fin_r & np.isfinite(y), np.abs(y - ref) > _old_f32_bar(ref, top), np.isfinite(y) != fin_r)
        clean_fails = old_fails(y0)
        for name, flag in ME.DEFECTS.items():
            _, _, xd, yd = ME.lane_frames(True, *args, defects=flag, libm_log=True)
            ok = np.isfinite(x0) & (x0 > 0) & np.isfinite(xd) & (xd > 0)
            with np.errstate(divide="ignore", invalid="ignore"):
                d = np.abs(np.log(xd[ok].astype(np.float64)) - np.log(x0[ok].astype(np.float64)))
                if d.size:
                    worst[name] = max(worst[name], float((d / ME.f32_bar(x0[ok])).max()))
                # a mismatch in which entries are finite, NaN or zero counts as caught outright
                if not np.array_equal(np.isnan(xd), np.isnan(x0)) or not np.array_equal(xd == 0, x0 == 0):
                    worst[name] = max(worst[name], np.inf)
                # the oracle comparison catches a defect where it rejects an entry that the clean kernel passes
                old_caught[name] |= bool((old_fails(yd) & ~clean_fails).any())
    print("\ndefect                 worst |d ln x| / float32 bar   caught by the oracle bar")
    for name in ME.DEFECTS:
        print(f"{name:22s} {worst[name]:16.3g}               {'yes' if old_caught[name] else 'NO (let through)'}")
    for name in ME.INVISIBLE:
        assert worst[name] == 0.0 and not old_caught[name], name
    missed = [k for k, v in worst.items() if not v > 2.0 and k not in ME.INVISIBLE]
    assert not missed, ("defects within twice the bar on every entry", missed, worst)
