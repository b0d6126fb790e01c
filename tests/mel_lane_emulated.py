"""mel512_kernel's log argument emulated on the host, the bars that hold the kernel to it, and the sweep that the CPU and
GPU tests of the emulation share (not a test module).

``tests/emul/mel_lane_emul.cpp`` runs ``mel_core.cuh`` lane by lane (the same FFT passes, lane tables, recombination and
pair rows the kernel runs) and forms each mel's band sum E as ``mel_dot_pairs`` does: the plan's packed, swizzled bands and
one ``fmaf`` chain over the band's bin quads in power-row order.  ``lane_frames`` returns per frame the power row 4|X_b|^2,
the band sums E and the log argument x (``max(E, floor)`` as Swift evaluates it, or ``E + floor``).

Float32 pairs (``Precision.f32``).  Every float32 operation of the device path up to the log is an explicit
``__fadd_rn`` / ``__fmul_rn`` / ``__fmaf_rn``, and the host build rounds the same operations the same way
(``-ffp-contract=off``), from the same lane tables (``load_lane_tables``).  So x is the device's log argument bit for bit,
and only the log is left: ``lg2.approx`` / ``__log2f`` times ln 2 in float32, 2^-22 absolute in log2 for arguments in
[0.5, 2] and 2 ulp elsewhere, which with the rounded ln 2 and the product gives (tests/mel_ex_restated.py, step 6)

    |y - ln x| <= 4u ln 2 + 6u |ln x|,   u = 2^-24, ln x in float64;   x = 0 gives -inf, x NaN gives NaN, x inf gives inf.

FP64 transform (``Precision.f64``).  Pre-emphasis and window are the same float32 operations on both sides (R_f = 0 in
mel_ex_restated.py's step 1); the two sides differ only where nvcc contracts a double multiply-add.  The bar restates
mel_ex_restated.py steps 2 to 6 for the difference of two evaluations, with S_f = sum_j |y_j w_j| over the frame:

2. Transform: 5 log2(512) 2^-53 per side on values of at most 4 S_f (the recombination's S and T reach 2 S_f each), counted
   twice, once per side: delta_T = 2 * 45 * 2^-53 * 4 S_f.  It holds for the radix-8 x 8 x 4 passes as for radix 2: every
   value of every pass is a partial DFT of the frame, and each pass adds at most 5 roundings of such values.
3. Re and Im of 2X rounded to float32 on each side: |xr_dev - xr_emu| <= delta_T + 2.01u (A + delta_T), A = |2X_b| taken
   from the emulated power as sqrt(p)(1 + 1.01u); the complex difference is at most D = sqrt(2) times that.
4. The power (three roundings on this path): |p_dev - p_emu| <= (2A + D) D + 2.01u ((A + D)^2 + A^2).
5. The band chain, the same 4 nq fmaf in the same order on both sides: |E_dev - E_emu| <= band + (4 nq + 1)u (2.01 E +
   band), band = sum_b w_b |p_dev - p_emu| over the mel's quad band.
6. The log: x_dev lies in [g(max(E - dE, 0)), g(E + dE)], g the floor rule (the additive floor's float32 add widens it by
   one rounding each way), and y = ln x_dev within 4u ln 2 + 6u |ln x_dev|.

Subnormal intermediates (the 1e-19 fixture with a log floor of 0) round absolutely: 2^-149 is added to each of steps 3 and
4 per bin and to step 5 per chain step, as mel_ex_restated.py does.

``DEFECTS`` names the emulator's defect flags, each one realistic kernel defect; the CPU tests show each moves some entry of
the sweep by more than twice the float32 bar (twice: a defective kernel's log may err toward the clean value by one bar).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
TINY = 2.0 ** -149
LN2 = float(np.log(2.0))
F32 = np.float32
BINS = 257
CENTER, PRE_PADDED, LEGACY = 0, 1, 2
TIME_MAJOR, MEL_MAJOR = 0, 1
TILE = 16

DEFECTS = {"twiddle_ulp": 1, "window_ulp": 2, "power_mul_add": 4, "dot_mul_add": 8, "tile_first_preemph": 16,
           "last_zero": 32, "no_swizzle": 64, "step_first_preemph": 128}
# A tile's pre-emphasised sample 0 feeds only buffer position 0 of the tile's first frame.  A window covers that position
# only when it starts there (a 512-sample window, or any window in the legacy placement), and then it meets the window's
# first coefficient, which for Hann is exactly 0 (symmetric and periodic alike): no output of the kernel depends on it.
INVISIBLE = ("tile_first_preemph",)

_LIB = None


def lib():
    """tests/emul/mel_lane_emul.cpp with fluidaudio_b200/csrc/mel_tables.cpp, compiled once per process into a temporary
    directory."""
    global _LIB
    if _LIB is not None:
        return _LIB
    csrc = os.path.join(ROOT, "fluidaudio_b200", "csrc")
    out = os.path.join(tempfile.mkdtemp(prefix="mel_lane_"), "libmel_lane.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I", csrc, "-I",
                           os.path.join(ROOT, "include"), "-o", out, os.path.join(ROOT, "tests", "emul", "mel_lane_emul.cpp"),
                           os.path.join(csrc, "mel_tables.cpp")])
    L = C.CDLL(out)
    f32p = np.ctypeslib.ndpointer(F32, flags="C_CONTIGUOUS")
    opt = C.c_void_p
    i32, i64, f32 = C.c_int, C.c_longlong, C.c_float
    L.mel_lane_frames.argtypes = [i32, f32p, i64, f32, i32, i32, i32, i32, f32, i32, f32p, f32p, f32, i32, i64, i32, opt,
                                  f32p, f32p, opt]
    L.mel_lane_dot.argtypes = [f32p, i64, i32, f32p, i32, f32, i32, f32p, f32p]
    _LIB = L
    return L


def _ptr(a):
    return None if a is None else a.ctypes.data


def lane_frames(f32: bool, audio, last, hop, window, off, pad, preemph, fb, floor, clamped, T, defects=0, power=False,
                libm_log=False):
    """(power [T x 257] or None, E [T x M], x [T x M], logf(x) [T x M] or None) of the emulated kernel."""
    audio = np.ascontiguousarray(audio, F32)
    fb = np.ascontiguousarray(fb, F32)
    window = np.ascontiguousarray(window, F32)
    M = fb.shape[0]
    P = np.zeros((T, BINS), F32) if power else None
    E = np.zeros((T, M), F32)
    x = np.zeros((T, M), F32)
    out = np.zeros((T, M), F32) if libm_log else None
    if T > 0:
        assert lib().mel_lane_frames(int(f32), audio, audio.size, F32(last), hop, window.size, off, pad, F32(preemph), M, fb,
                                     window, F32(floor), int(clamped), T, defects, _ptr(P), E, x, _ptr(out)) == 0
    return P, E, x, out


def lane_dot(power, fb, floor=0.0, clamped=0, defects=0):
    """(E, x) [rows x M] of the filterbank stage alone on power rows [rows x 257] in bin order."""
    power = np.ascontiguousarray(power, F32)
    fb = np.ascontiguousarray(fb, F32)
    rows, M = power.shape[0], fb.shape[0]
    E, x = np.zeros((rows, M), F32), np.zeros((rows, M), F32)
    assert lib().mel_lane_dot(power, rows, M, fb, defects, F32(floor), int(clamped), E, x) == 0
    return E, x


def quad_bands(fb):
    """Each mel's band as the plan packs it: [lo, hi) rounded out to bin quads, (0, 0) when empty."""
    M = fb.shape[0]
    lo, hi = np.zeros(M, np.int64), np.zeros(M, np.int64)
    for m in range(M):
        nz = np.flatnonzero(fb[m])
        if nz.size:
            lo[m], hi[m] = nz[0] & ~3, (nz[-1] + 4) & ~3
    return lo, hi


# ================================================================================================ bars
def f32_bar(x):
    """Bar on |y - ln x| for the float32-pair path (finite, non-zero x)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return 4 * U * LN2 + 6 * U * np.abs(np.log(np.asarray(x, np.float64)))


def check_f32(y, x, what):
    """Float32 pairs: y [T x M] the device's output, x the emulated log argument.  Returns the worst |y - ln x| / bar."""
    y = np.asarray(y, np.float32)
    x = np.asarray(x, np.float32)
    assert y.shape == x.shape, (what, y.shape, x.shape)
    nan = np.isnan(x)
    assert np.array_equal(np.isnan(y), nan), (what, "NaN pattern", np.argwhere(np.isnan(y) != nan)[:4])
    zero = x == 0
    assert (y[zero] == -np.inf).all(), (what, "log 0")
    inf = np.isinf(x)
    assert (y[inf] == np.inf).all(), (what, "log inf")
    use = ~(nan | zero | inf)
    if not use.any():
        return 0.0
    xv = x[use].astype(np.float64)
    d = np.abs(y[use].astype(np.float64) - np.log(xv))
    frac = d / f32_bar(xv)
    worst = float(frac.max())
    assert worst <= 1.0, (what, worst, "at", np.argwhere(use)[int(frac.argmax())], "y", float(y[use][frac.argmax()]),
                          "x", float(xv[frac.argmax()]))
    return worst


def frame_abs_sums(audio, last, hop, window, off, pad, preemph, T):
    """S_f = sum_j |y_j w_j| over each frame, bounded above with |y_i| <= |x_i| + |a| |x_{i-1}| (x_{-1} = last)."""
    x = np.abs(np.asarray(audio, np.float64))
    prev = np.concatenate([[abs(float(F32(last)))], x[:-1]]) if x.size else x
    yb = x + abs(float(F32(preemph))) * prev
    w = np.abs(np.asarray(window, np.float64))
    need = (T - 1) * hop + 512
    buf = np.zeros(need + pad + 1)
    n = min(yb.size, need - 0)
    buf[pad:pad + n] = yb[:n]
    view = np.lib.stride_tricks.sliding_window_view(buf[off:off + (T - 1) * hop + w.size], w.size)[::hop][:T]
    return (view @ w) * 1.01


def check_f64(y, E, x, power, S, fb, floor, clamped, what):
    """FP64 transform: y [T x M] against the emulated E / x / power [T x 257] and S_f [T], within the bar of the module
    docstring.  Returns the worst deviation as a fraction of the bar (toward whichever side y lies)."""
    y = np.asarray(y, np.float32).astype(np.float64)
    nan = np.isnan(x)
    assert np.array_equal(np.isnan(y), nan), (what, "NaN pattern", np.argwhere(np.isnan(y) != nan)[:4])
    lo_b, hi_b = quad_bands(fb)
    nq = (hi_b - lo_b) // 4
    w = np.asarray(fb, np.float64) * 0.25
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        p = power.astype(np.float64)
        A = np.sqrt(p) * (1 + 1.01 * U)
        dT = 2 * 45 * 2.0 ** -53 * 4 * S[:, None]
        D = np.sqrt(2.0) * (dT + 2.01 * U * (A + dT) + 2 * TINY)
        dp = (2 * A + D) * D + 2.01 * U * ((A + D) ** 2 + A ** 2) + 8 * TINY
        Ed = E.astype(np.float64)
        band = np.zeros_like(Ed)
        for m in range(w.shape[0]):
            if hi_b[m] > lo_b[m]:
                s = slice(lo_b[m], min(hi_b[m], BINS))
                band[:, m] = dp[:, s] @ w[m, s]
        dE = band + (4 * nq + 1) * (U * (2.01 * Ed + band) + 2 * TINY)
        fl = float(F32(floor))
        if clamped:
            lo = np.log(np.maximum(np.maximum(Ed - dE, 0.0), fl))
            hi = np.log(np.maximum(Ed + dE, fl))
        else:
            lo = np.log(np.maximum(Ed - dE, 0.0) + fl) + np.log1p(-U)
            hi = np.log(Ed + dE + fl) + np.log1p(U)
        mag = np.maximum(np.where(np.isfinite(lo), np.abs(lo), 0.0), np.where(np.isfinite(hi), np.abs(hi), 0.0))
        err = 4 * U * LN2 + 6 * U * mag
        lo, hi = lo - err, hi + err
        hi = np.where(Ed + dE > np.finfo(np.float32).max, np.inf, hi)   # the device's power may overflow where ours did not
        use = ~nan
        yv, xl = y[use], np.log(x[use].astype(np.float64))
        ok = (yv >= lo[use]) & (yv <= hi[use])
        ok |= (yv == xl)                       # equal, infinities included
        assert ok.all(), (what, "outside the bar at", np.argwhere(use)[np.flatnonzero(~ok)[:4]], yv[~ok][:4], xl[~ok][:4],
                          lo[use][~ok][:4], hi[use][~ok][:4])
        fin = np.isfinite(xl) & np.isfinite(yv) & (yv != xl)
        up = np.where(yv > xl, (yv - xl) / (hi[use] - xl), (xl - yv) / (xl - lo[use]))
        return float(up[fin].max()) if fin.any() else 0.0


# ================================================================================================ the sweep
WINS = (512, 449, 448, 400, 385, 384, 383, 256, 64)
MELS = (1, 3, 23, 40, 81, 128, 200, 257, 512)
RATES = (8000, 16000, 22050, 48000)
FLOORS = (2.0 ** -24, 1e-10, 1e-38, 0.0)
FRAMES = (1, 2, 15, 16, 17, 31, 33)
HOPS = (160, 2, 64, 128, 158, 256, 320, 512, 514, 576)
SIGNALS = ("tone_noise", "speech", "square", "dc", "tiny", "huge", "tiny_square")


def signal(kind: str, n: int, seed: int, sr: int = 16000) -> np.ndarray:
    """tone + noise, speech-like (60 dB range), a +-1 square wave and a DC of 0.25 (exact spectra), tone + noise at 1e-19
    and a square wave of +-3e-19 (subnormal power) and tone + noise with its middle third at 1e18 (power overflowing inside quad-rounded bands)."""
    from fluidaudio_b200 import synth
    if kind == "tone_noise":
        return synth.tone_noise_audio(n, seed=seed)
    if kind == "speech":
        return synth.speech_like_audio(n, seed=seed, sample_rate=sr)
    if kind == "square":
        return np.where((np.arange(n) // (16 + seed % 48)) % 2 == 0, 1.0, -1.0).astype(F32)
    if kind == "dc":
        return np.full(n, 0.25, F32)
    if kind == "tiny":
        return (synth.tone_noise_audio(n, seed=seed) * F32(1e-19)).astype(F32)
    if kind == "tiny_square":
        return np.where((np.arange(n) // (16 + seed % 48)) % 2 == 0, 3e-19, -3e-19).astype(F32)
    if kind == "huge":
        x = synth.tone_noise_audio(n, seed=seed)
        x[n // 3:2 * n // 3] *= F32(1e18)
        return x
    raise ValueError(kind)


def length_for(frames, hop, win, mode):
    """A sample count whose frame count in ``mode`` is about ``frames``."""
    if mode == CENTER:
        return max(1, (frames - 1) * hop + win - 512 + 1)
    if mode == PRE_PADDED:
        return (frames - 1) * hop + 512
    return (frames - 1) * hop + win


def cross_cases():
    """Window x sample rate x floor mode x log floor, with the mel count, hop, pre-emphasis (0.97 or 0: the plain copy
    path), frame count, signal and padding mode dealt round robin.  Every mel count of MELS meets every rate."""
    out = []
    i = 0
    for win in WINS:
        for sr in RATES:
            for clamped in (0, 1):
                for fl in FLOORS:
                    i += 1
                    out.append(dict(win=win, sr=sr, clamped=clamped, floor=fl, n_mels=MELS[(i + i // 9) % len(MELS)],
                                    hop=HOPS[i % len(HOPS)], preemph=0.0 if i % 5 == 2 else 0.97,
                                    frames=FRAMES[i % len(FRAMES)], signal=SIGNALS[i % len(SIGNALS)],
                                    mode=(CENTER, PRE_PADDED, LEGACY)[i % 3], last=(0.3, -0.45, 0.7)[i % 3], seed=i))
    # subnormal power at every mel count under a log floor of 0 (the __log2f path): the only inputs where a power or band
    # sum rounded once more than the kernel rounds it moves the log by more than the log's own error.  Even there it takes a
    # band dominated by a few-ulp subnormal bin: the +-3e-19 square wave of period 19 (seed 3) at 512 mels has such bands.
    for j, nm in enumerate(MELS):
        for sig in ("tiny", "tiny_square"):
            i += 1
            out.append(dict(win=400, sr=(16000, 48000)[j % 2], clamped=i % 2, floor=0.0, n_mels=nm, hop=160, preemph=0.97,
                            frames=33, signal=sig, mode=CENTER, last=0.3, seed=3 + 48 * j))
    return out


def placement(cfg, mode):
    """(window offset, centre pad, pre-emphasis) of a call in ``mode``."""
    off = 0 if mode == LEGACY else (512 - cfg["win"]) // 2
    pad = 256 if mode == CENTER else 0
    pre = 0.0 if mode == LEGACY else cfg["preemph"]
    return off, pad, pre


def frame_count(n, hop, win, mode):
    """MelPlan::frame_count (C++ division truncates toward zero)."""
    div = lambda a: a // hop if a >= 0 else -(-a // hop)
    if mode == CENTER:
        return 1 + div(n + 512 - win)
    if mode == PRE_PADDED:
        return max(0, div(n - 512) + 1)
    return 1 + div(n - win)
