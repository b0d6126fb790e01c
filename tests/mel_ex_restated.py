"""A float64 restatement of an ex handle's log-mel, its derived per-entry bar and the configuration sweep that the CPU and
GPU tests of the torch-style frontends share (not a test module).

``restate`` takes a handle's configuration (``Cfg``) and the handle's own window and table (``fa_mel_get_window`` /
``fa_mel_get_filterbank`` on the GPU, ``mt_tables`` of tests/emul/mel_tables_shim.cpp on the CPU; both are pinned bit for
bit to the oracle) and computes [T x nMels] in float64:

* framing per mode: ``.center`` pads nFFT/2 zeros, or on a reflect handle reads the reference's clamped reflection
  (index i < 0 reads x[min(-i, n-1)], i >= n reads x[max(2n-2-i, 0)], an empty clip reads zeros); ``.prePadded`` reads
  the clip as it is; legacy ``compute()`` puts the window at offset 0 instead of (nFFT - win) / 2;
* pre-emphasis y[i] = x[i] - a x[i-1] with ``last`` standing for x[-1] (none on a reflect handle, none in legacy mode);
* the window product, ``numpy.fft.rfft`` in float64, |X|^p, each mel's band of the table (a mel whose filter is empty
  reads nothing: its value is 0, as in the kernels), log(E + floor) or log(max(E, floor)), then (L - mean) / std.

It also returns what the bar needs: S_f = sum_j |y_j w_j| per frame, |X_b|, E_m and each mel's band in quads.

The bar, per output entry, with u = 2^-24, from the operations of ``mel_generic_kernel`` (mel_kernels.cu):

1. Pre-emphasis and window: ``fmaf`` (one rounding), then ``__fmul_rn``: <= 2u |y_j w_j| per sample.  Sample 0 rounds
   a * last and the difference separately (``preemph_first``), so S_f holds |a last w_j| for it as well.  Without
   pre-emphasis the frame is one float32 product of two float32 values, exact in float64, so R_f takes the rounding
   that product actually makes instead of its bound u |x_j w_j| (zero for a +-1 square wave or a DC of 0.25).  With
   it, R_f = 2.01u S_f.
2. FFT: FP64 radix-2 with a float64 twiddle table, c log2(n) 2^-53 S_f with c = 5 (negligible beside step 1, stated).
3. Re and Im rounded to float32: u |X_b|.  Steps 1-3: delta_b <= R_f + u |X_b| (+ step 2), as every input error
   reaches a bin with weight |W^k| = 1 (the 0.01 absorbs second-order terms).
4. Power ``pw = xr*xr + xi*xi`` in three roundings: relative 2.01u.  Then
   |X|^2: 2|X| delta + delta^2 + 2.01u (|X| + delta)^2 (the tile holds 4 pw, the weights 1/4: exact scalings);
   |X|:   dm = delta + 2.01u (|X| + delta), ``__fsqrt_rn`` halving pw's relative error and adding one rounding;
   |X|^p: the interval [max(|X| - dm, 0), |X| + dm] through t^p, plus ``powf``'s documented 4 ulp, 8u (|X| + dm)^p.
5. Band product: a chain of 4 nq ``fmaf`` over non-negative terms (explicit zero weights included): (4 nq + 1)u E~,
   E~ = E + the band sum of step 4's errors.  The same bound covers the oracle's rounded products and sums.
6. Log: the interval [max(E - dE, 0), E + dE] through log(. + floor) or log(max(., floor)), plus 1.01u for the
   additive floor's float32 add.  The device log is ``__log2f`` (``lg2.approx.f32``) times ln 2 in float32: 2^-22
   absolute in log2 for arguments in [0.5, 2], 2 ulp of the result elsewhere.  Taken together as
   2^-22 (1 + |log2 x|), times ln 2, plus 2u |L| for the rounded ln 2 and the product: 4u ln 2 + 6u |L|.  The
   absolute term is there because near an argument of 1 the log is near 0 and its error is not relative.
7. Affine: (|dL| + u |L - mean|) / |std| + 1.01u |out|.

Steps 3 to 5 are relative bounds, which hold for normal float32 values.  Where they reach the subnormal range (a log
floor of 0 with |X|^2 or |X|^p below 2^-126) a rounding errs by up to 2^-150 absolute instead, so the bar adds
2^-149 to delta_b, 8 * 2^-149 per bin to step 4 and (4 nq + 1) 2^-149 to step 5.

Only two figures come from documentation rather than derivation: ``powf``'s 4 ulp (CUDA C++ Programming Guide 12.x,
"Mathematical Functions", single-precision table) and ``lg2.approx.f32`` / ``__log2f``'s 2^-22 absolute error in
[0.5, 2] and 2 ulp elsewhere (PTX ISA 8.x, ``lg2``; CUDA Math API 12.x, single-precision intrinsics).

The bar is loose in weak bins, where S_f >> |X_b|, by design; in a frame's strongest band it is tight.  There the
model gives dE / E <= 4.02u S_f sqrt(sum_b w_b / E) + (4 nq + 5)u; for white noise S_f / |X| ~ sqrt(nFFT), which is
about 4u sqrt(nFFT): 1.5e-5 at nFFT 4096, 5e-6 at 512.  ``strong_ceiling`` states the ceiling the tests assert there.

``Cfg.from_ex`` reads a ``fa_mel_ex_config``; ``sweep_configs`` deals the sweep's configurations round robin so that
every (kReflect, kSpectrum, kAffine) variant of the generic kernel gets at least three.
"""
from __future__ import annotations

import ctypes as C
import itertools
import os
import subprocess
from dataclasses import dataclass, replace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
TINY = 2.0 ** -149   # the smallest float32 subnormal: twice the absolute rounding error of any subnormal result
LN2 = float(np.log(2.0))
F32 = np.float32
CENTER, PRE_PADDED, LEGACY = 0, 1, 2
FB_AUDIO_MEL, FB_COHERE, FB_STYLETTS2, FB_LUXTTS = 0, 1, 2, 3
SPEC_POWER, SPEC_MAGNITUDE, SPEC_GENERAL = 0, 1, 2
MUTATIONS = ("window_shift", "torch_reflect", "preemph_reflect", "power2", "affine_order", "band_shift", "f32_fft")


@dataclass(frozen=True)
class Cfg:
    sample_rate: int = 16000
    n_mels: int = 128
    n_fft: int = 512
    hop: int = 160
    win: int = 400
    preemph: float = 0.97
    pad_to: int = 1
    floor: float = 2.0 ** -24
    clamped: bool = False
    periodic: bool = False
    kind: int = FB_AUDIO_MEL
    filter_sr: int = 0
    f_min: float = 0.0
    f_max: float = 0.0
    reflect: bool = False
    power: float = 2.0
    mean: float = 0.0
    std: float = 1.0

    @staticmethod
    def from_ex(ex) -> "Cfg":
        b = ex.base
        return Cfg(b.sample_rate, b.n_mels, b.n_fft, b.hop_length, b.win_length, float(F32(b.preemph)), max(1, b.pad_to),
                   float(F32(b.log_floor)), bool(b.log_floor_mode), bool(b.window_periodic), ex.filterbank,
                   ex.filter_sample_rate, float(F32(ex.f_min)), float(F32(ex.f_max)), ex.center_edge == 1,
                   float(F32(ex.spectrum_power)), float(F32(ex.log_mean)), float(F32(ex.log_std)))

    def ex_fields(self) -> dict:
        """Keyword arguments of ``fluidaudio_b200.mel.ex_config(None, ...)`` for this configuration."""
        return dict(sample_rate=self.sample_rate, n_mels=self.n_mels, n_fft=self.n_fft, hop_length=self.hop,
                    win_length=self.win, preemph=self.preemph, pad_to=self.pad_to, log_floor=self.floor,
                    log_floor_mode=int(self.clamped), window_periodic=int(self.periodic), filterbank=self.kind,
                    filter_sample_rate=self.filter_sr, f_min=self.f_min, f_max=self.f_max,
                    center_edge=int(self.reflect), spectrum_power=self.power, log_mean=self.mean, log_std=self.std)

    @property
    def spectrum(self) -> int:
        p = float(F32(self.power))
        return SPEC_POWER if p == 2.0 else (SPEC_MAGNITUDE if p == 1.0 else SPEC_GENERAL)

    @property
    def affine(self) -> bool:
        return float(F32(self.mean)) != 0.0 or float(F32(self.std)) != 1.0

    def variant(self, mode: int) -> tuple:
        """(kReflect, kSpectrum, kAffine) of the generic kernel a call in ``mode`` launches (MelPlan::launch): reflection
        only for ``.center`` on a reflect handle; the handle's other modes run the non-reflect twin."""
        return (self.reflect and mode == CENTER, self.spectrum, self.affine)

    def generic(self) -> bool:
        """Does the handle take mel_generic_kernel (MelPlan::init)?  Otherwise mel512_kernel, which a sweep handle reaches
        only at nFFT 512, an even hop <= 1024, |X|^2, no reflection and no affine step (and shared memory that fits)."""
        return (self.n_fft != 512 or self.hop % 2 == 1 or self.hop > 1024 or self.reflect or self.spectrum != SPEC_POWER
                or self.affine)


def c_div(a: int, b: int) -> int:
    """C++ integer division (truncates toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def frame_count(cfg: Cfg, n: int, mode: int) -> int:
    """MelPlan::frame_count and the "empty" guard: 0 frames when the library returns its zero row."""
    if n <= 0:
        return 0
    if mode == CENTER:
        T = 1 + c_div(n + 2 * (cfg.n_fft // 2) - cfg.win, cfg.hop)
    elif mode == PRE_PADDED:
        T = max(0, c_div(n - cfg.n_fft, cfg.hop) + 1)
    else:
        T = 1 + c_div(n - cfg.win, cfg.hop)
    return max(T, 0)


def reflect_clamped(i: np.ndarray, n: int) -> np.ndarray:
    """The reference's reflectPad clamps, from the rule in include/fluidaudio_b200.h."""
    return np.where(i < 0, np.minimum(-i, n - 1), np.where(i >= n, np.maximum(2 * n - 2 - i, 0), i))


def bands(fb: np.ndarray):
    """Each mel's band as the kernels pack it: [lo, hi) quad-aligned around its non-zero weights, (0, 0) when empty.
    test_mel_ex_restated.py holds it to the packer's own (``packed_bands``) on every table of the sweep."""
    M = fb.shape[0]
    lo, hi = np.zeros(M, np.int64), np.zeros(M, np.int64)
    for m in range(M):
        nz = np.flatnonzero(fb[m])
        if nz.size:
            lo[m], hi[m] = nz[0] & ~3, (nz[-1] + 4) & ~3
    return lo, hi


@dataclass
class Restated:
    out: np.ndarray     # [T x M] the handle's output
    L: np.ndarray       # [T x M] the log before the affine step
    E: np.ndarray       # [T x M] mel values
    S: np.ndarray       # [T] sum_j |y_j w_j| (+ the extra pre-emphasis terms)
    R: np.ndarray       # [T] bound on sum_j |error of the float32 frame sample j| (steps 1 of the bar)
    absX: np.ndarray    # [T x bins]
    nq: np.ndarray      # [M] band width in quads
    fb: np.ndarray      # [M x bins] float64 table
    lo: np.ndarray
    hi: np.ndarray


def restate(cfg: Cfg, window, fb, audio, mode: int = CENTER, last: float = 0.0, T: int | None = None,
            mutate: str | None = None, preemph_two_roundings: bool = False) -> Restated:
    """The handle's log-mel of ``audio`` in float64, T frames (default: the library's count for ``mode``).
    ``mutate`` (one of MUTATIONS) restates a defect instead, for the tests that show the bar catches it.
    ``preemph_two_roundings``: the bar's S_f also covers a pre-emphasis that rounds a x[i-1] before subtracting (the
    Cohere oracle)."""
    x = np.asarray(audio, F32).astype(np.float64)
    n = x.size
    n_fft, win = cfg.n_fft, cfg.win
    bins = n_fft // 2 + 1
    if T is None:
        T = frame_count(cfg, n, mode)
    w = np.asarray(window, np.float64).reshape(-1)
    fb64 = np.asarray(fb, np.float64).copy()
    off = 0 if mode == LEGACY else (n_fft - win) // 2
    if mutate == "window_shift":
        off = off + 1 if off + 1 + win <= n_fft else off - 1
    pad = n_fft // 2 if mode == CENTER else 0
    reflect = cfg.reflect and mode == CENTER
    a = 0.0 if mode == LEGACY else float(F32(cfg.preemph))
    if mutate == "preemph_reflect" and reflect:
        a = 0.97
    # pre-emphasised signal (exact), and the magnitude of the rounded product a x[i-1] per sample
    prev = np.concatenate([[float(F32(last))], x[:-1]]) if n else x
    y = x - a * prev if a != 0.0 else x
    extra = np.abs(a * prev) if a != 0.0 else np.zeros(n)
    if a != 0.0 and not preemph_two_roundings and n:
        extra = np.concatenate([extra[:1], np.zeros(n - 1)])   # only sample 0 rounds twice in the kernel
    j = off + np.arange(win)
    fb_use = fb64
    if mutate == "band_shift":
        fb_use = fb64.copy()
        for m in range(fb_use.shape[0]):
            nz = np.flatnonzero(fb_use[m])
            if nz.size > 1:
                fb_use[m, nz[0]] = 0.0
    lo, hi = bands(fb64)
    nq = (hi - lo) // 4
    E = np.zeros((T, fb64.shape[0]))
    S = np.zeros(T)
    R = np.zeros(T)
    absX = np.zeros((T, bins))
    p = 2.0 if mutate == "power2" else float(F32(cfg.power))
    step = max(1, (1 << 22) // n_fft)
    for f0 in range(0, T, step):
        f = np.arange(f0, min(T, f0 + step))
        i = f[:, None] * cfg.hop - pad + j[None, :]
        if reflect:
            if n == 0:
                v, e = np.zeros(i.shape), np.zeros(i.shape)
            else:
                if mutate == "torch_reflect":
                    r = np.pad(np.arange(n), n_fft // 2 + 1, mode="reflect")[i + n_fft // 2 + 1]
                else:
                    r = reflect_clamped(i, n)
                src = y if mutate == "preemph_reflect" else x
                v, e = src[r], (extra[r] if mutate == "preemph_reflect" else np.zeros(i.shape))
        else:
            inside = (i >= 0) & (i < n)
            ic = np.clip(i, 0, max(n - 1, 0))
            v = np.where(inside, y[ic] if n else 0.0, 0.0)
            e = np.where(inside, extra[ic] if n else 0.0, 0.0)
        frame = np.zeros((f.size, n_fft))
        frame[:, j] = v * w[None, :]
        with np.errstate(invalid="ignore", over="ignore"):
            S[f] = (np.abs(v) + e) @ np.abs(w)
            if a == 0.0:   # the samples are the float32 input: the product's rounding is known exactly
                R[f] = np.abs((v * w[None, :]).astype(F32).astype(np.float64) - v * w[None, :]).sum(1)
            else:
                R[f] = 2.01 * U * S[f]
        if mutate == "f32_fft":
            import scipy.fft
            X = scipy.fft.rfft(frame.astype(F32), axis=1).astype(np.complex128)
        else:
            X = np.fft.rfft(frame, axis=1)
        ax = np.abs(X)
        absX[f] = ax
        with np.errstate(invalid="ignore", over="ignore"):
            spec = X.real ** 2 + X.imag ** 2 if p == 2.0 else ax ** p
            for m in range(fb64.shape[0]):
                if hi[m] > lo[m]:
                    E[f, m] = spec[:, lo[m]:min(hi[m], bins)] @ fb_use[m, lo[m]:min(hi[m], bins)]
    fl = float(F32(cfg.floor))
    with np.errstate(divide="ignore", invalid="ignore"):
        L = np.log(np.maximum(E, fl)) if cfg.clamped else np.log(E + fl)
        L = np.where(np.isnan(E), np.nan, L)
        mean, std = float(F32(cfg.mean)), float(F32(cfg.std))
        out = L / std - mean if mutate == "affine_order" else (L - mean) / std
    return Restated(out, L, E, S, R, absX, nq, fb64, lo, hi)


def bar(cfg: Cfg, r: Restated, f32_transform: bool = False) -> tuple[np.ndarray, np.ndarray]:
    """(bar on the output, bar on the log before the affine step), [T x M] each; see the module docstring.
    ``f32_transform``: the transform is mel512_kernel's float32 FFT (FA_MEL_PRECISION_F32) instead of FP64.  Every
    entry of every radix-2 stage is a partial DFT of the frame, so its magnitude is at most S_f; a stage's twiddle
    product (two float32 products and an add per component, float32 twiddles within u) and its butterfly add put at
    most 5u S_f into each entry, so the transform term becomes 5u log2(nFFT) S_f in delta_b."""
    n_fft = cfg.n_fft
    p = float(F32(cfg.power))
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        ax = r.absX
        S = r.S[:, None]
        d = r.R[:, None] + U * ax + 5 * np.log2(n_fft) * (U if f32_transform else 2.0 ** -53) * S + TINY
        if p == 2.0:
            dspec = 2 * ax * d + d * d + 2.01 * U * (ax + d) ** 2
        else:
            dm = d + 2.01 * U * (ax + d)
            if p == 1.0:
                dspec = dm
            else:
                top = (ax + dm) ** p
                dspec = np.maximum(top - ax ** p, ax ** p - np.maximum(ax - dm, 0.0) ** p) + 8 * U * top
        dspec = dspec + 8 * TINY
        T, M = r.E.shape
        dE = np.zeros((T, M))
        for m in range(M):
            if r.hi[m] > r.lo[m]:
                s = slice(r.lo[m], min(r.hi[m], ax.shape[1]))
                band = dspec[:, s] @ r.fb[m, s]
                dE[:, m] = band + (4 * r.nq[m] + 1) * (U * (r.E[:, m] + band) + TINY)
        fl = float(F32(cfg.floor))
        E = r.E
        hi, lo = E + dE, np.maximum(E - dE, 0.0)
        g = (lambda v: np.log(np.maximum(v, fl))) if cfg.clamped else (lambda v: np.log(v + fl))
        gE = g(E)
        dL = np.maximum(g(hi) - gE, gE - g(lo))
        dL = np.where(np.isfinite(gE), dL, 0.0)
        dL = dL + (0.0 if cfg.clamped else 1.01 * U) + 4 * U * LN2 + 6 * U * (np.abs(np.where(np.isfinite(gE), gE, 0.0))
                                                                             + dL)
        mean, std = float(F32(cfg.mean)), float(F32(cfg.std))
        if not cfg.affine:
            return dL, dL
        Lm = np.where(np.isfinite(r.L), r.L, 0.0)
        dout = (dL + U * np.abs(Lm - mean)) / abs(std) + 1.01 * U * np.abs((Lm - mean) / std)
    return dout, dL


def strong_ceiling(cfg: Cfg, r: Restated, rows) -> np.ndarray:
    """The ceiling asserted for the log-domain bar at each frame's strongest mel (``rows``: (frame, mel) index arrays):
    16u sqrt(nFFT) for the transform (4.02u S_f sqrt(sum w / E), with S_f / |X| ~ sqrt(nFFT) and a factor 4 of room for
    windowed speech), (4 nq + 8)u for the band product, the power and the log's adds, and the log's 4u ln 2 + 6u |L|."""
    f, m = rows
    return 16 * U * np.sqrt(cfg.n_fft) + (4 * r.nq[m] + 8) * U + 4 * U * LN2 + 6 * U * np.abs(r.L[f, m])


def strongest(r: Restated, floor: float):
    """(frame, mel) of each frame's strongest mel whose value is well above the floor (1e3 floor, and > 0)."""
    E = np.where(np.isfinite(r.E), r.E, -1.0)
    m = E.argmax(1)
    f = np.arange(E.shape[0])
    keep = (E[f, m] > max(1e3 * floor, 0.0)) & (E[f, m] > 0)
    return f[keep], m[keep]


def compare(got, cfg: Cfg, r: Restated, what, f32_transform: bool = False):
    """Worst |d| / bar of ``got`` [T x M] against the restatement; raises on an entry outside the bar, on a non-finite
    entry where the restatement is finite with a finite bar, and on a finite one where it is not finite."""
    got = np.asarray(got, np.float64)
    b, _ = bar(cfg, r, f32_transform)
    ref = r.out
    fin_r = np.isfinite(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), (what, "NaN pattern")
    inf_r = np.isinf(ref)
    assert np.array_equal(got[inf_r], ref[inf_r]), (what, "infinities")
    bad = fin_r & ~np.isfinite(got) & np.isfinite(b)
    assert not bad.any(), (what, "non-finite where the restatement is finite", np.argwhere(bad)[:4])
    use = fin_r & np.isfinite(got)
    if not use.any():
        return 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        frac = np.abs(got[use] - ref[use]) / b[use]
    frac = np.where(np.abs(got[use] - ref[use]) == 0, 0.0, frac)
    worst = float(frac.max())
    assert worst <= 1.0, (what, worst, np.argwhere(use)[int(frac.argmax())])
    return worst


# ================================================================================================ the sweep
NFFTS = (32, 64, 256, 512, 1024, 2048, 4096)
MELS = (1, 3, 80, 128, 257, 512)
POWERS = {SPEC_POWER: (2.0,), SPEC_MAGNITUDE: (1.0,), SPEC_GENERAL: (0.5, 1.5, 3.0)}
FLOORS = ((False, 1e-5), (True, 2.0 ** -24), (False, 1e-10), (True, 0.0), (False, 0.0), (True, 1e-5),
          (False, 2.0 ** -24), (True, 1e-10))
AFFINE = ((-4.0, 4.0), (1.5, -0.37))
RATES = (8000, 16000, 22050, 24000, 44100, 48000)
VARIANTS = [(rf, sp, af) for rf in (False, True) for sp in (SPEC_POWER, SPEC_MAGNITUDE, SPEC_GENERAL)
            for af in (False, True)]


def sweep_configs(per_variant: int = 4):
    """Handles for every generic-kernel variant, ``per_variant`` each, the other axes dealt round robin: table kind
    (Cohere with f_min / f_max variants, StyleTTS2 with filter rates 16000 / 22050 / 24000), nFFT, window (nFFT,
    nFFT - 1, nFFT/2 + 1, 1), hop (1, odd, even, = win, > nFFT), mels, p, log floor, (mean, std), rate and pad_to."""
    k = itertools.count()
    out = []
    for rep in range(per_variant):
        for vi, (rf, sp, af) in enumerate(VARIANTS):
            i = next(k)
            kind = i % 4
            n_fft = NFFTS[(i + rep) % len(NFFTS)]
            win = [n_fft, n_fft - 1, n_fft // 2 + 1, 1][(i // 3 + rep) % 4]
            hop = [1, 2 * (i % 50) + 37, 2 * (i % 40) + 160, win, n_fft + 3 + 2 * (i % 5)][(i // 3 + rep) % 5]
            if hop == 1 and n_fft > 256:
                hop = 3   # hop 1 stays with small transforms: its short clips still cover the sweep's lengths
            sr = RATES[(i // 2) % len(RATES)]
            clamped, floor = FLOORS[i % len(FLOORS)]
            p = POWERS[sp][(i // 12) % len(POWERS[sp])]
            mean, std = AFFINE[i % 2] if af else (0.0, 1.0)
            periodic = (i % 3 == 0) or (win == 1 and kind != FB_COHERE)
            f_min = f_max = 0.0
            filter_sr = 0
            if kind == FB_COHERE:
                f_min, f_max = [(0.0, 0.0), (20.0, 0.0), (125.0, 0.3 * sr), (0.0, sr / 2)][(i // 4) % 4]
            elif kind == FB_STYLETTS2:
                filter_sr = (16000, 22050, 24000)[(i // 4) % 3]
            out.append(Cfg(sample_rate=sr, n_mels=MELS[(i + 2 * rep) % len(MELS)], n_fft=n_fft, hop=hop, win=win,
                           preemph=0.0 if rf or i % 4 == 1 else 0.97, pad_to=(1, 3)[i % 2], floor=floor,
                           clamped=clamped, periodic=periodic, kind=kind, filter_sr=filter_sr, f_min=f_min,
                           f_max=f_max, reflect=rf, power=p, mean=mean, std=std))
    return out


def clip_lengths(cfg: Cfg, rate: int):
    """0, 1, 2, nFFT/2 - 1 .. + 1, nFFT - 1, nFFT, 5 hops +- 1 and about 2 s (hop 1 and nFFT 4096 stop at 8 hops)."""
    h, n = cfg.hop, cfg.n_fft
    base = {0, 1, 2, n // 2 - 1, n // 2, n // 2 + 1, n - 1, n, 5 * h - 1, 5 * h + 1}
    long = 2 * rate + 17 if (h > 4 and n < 4096) else n + 8 * h + 5
    return sorted(v for v in base | {long} if v >= 0)


def signal(kind: str, n: int, rate: int, seed: int = 0) -> np.ndarray:
    """noise, speech (synth.speech_like_audio), tone (on a bin centre over -100 dB noise), silence, dc, square
    (clipped)."""
    from fluidaudio_b200 import synth
    rng = np.random.default_rng(seed * 7919 + n)
    t = np.arange(n)
    if kind == "noise":
        return (rng.standard_normal(n) * 0.3).astype(F32)
    if kind == "speech":
        return synth.speech_like_audio(n, sample_rate=rate) if n else np.zeros(0, F32)
    if kind == "tone":
        return (0.5 * np.sin(2 * np.pi * 37 * t / 512) + 1e-5 * rng.standard_normal(n)).astype(F32)
    if kind == "silence":
        return np.zeros(n, F32)
    if kind == "dc":
        return np.full(n, 0.25, F32)
    if kind == "square":
        return np.clip(3.0 * np.sign(np.sin(2 * np.pi * 5 * t / rate + 0.1)), -1.0, 1.0).astype(F32)
    raise ValueError(kind)


SIGNALS = ("noise", "speech", "tone", "silence", "dc", "square")


# ================================================================================================ CPU tables
def mel_tables_lib(outdir: str):
    """tests/emul/mel_tables_shim.cpp with fluidaudio_b200/csrc/mel_tables.cpp, compiled with g++ into ``outdir``: the
    plan's host tables, packing, window placement and ex config check (test_mel_tables.py uses every entry point)."""
    csrc = os.path.join(ROOT, "fluidaudio_b200", "csrc")
    out = os.path.join(outdir, "libmel_tables.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I", csrc, "-I",
                           os.path.join(ROOT, "include"), "-o", out,
                           os.path.join(ROOT, "tests", "emul", "mel_tables_shim.cpp"), os.path.join(csrc, "mel_tables.cpp")])
    L = C.CDLL(out)
    f32p = np.ctypeslib.ndpointer(F32, flags="C_CONTIGUOUS")
    i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
    u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
    i32, f32 = C.c_int32, C.c_float
    L.mt_tables.argtypes = [i32, i32, i32, i32, i32, i32, i32, f32, f32, f32p, f32p]
    L.mt_pack_sizes.argtypes = [f32p, i32, i32, C.POINTER(i32), C.POINTER(i32)]
    L.mt_pack.argtypes = [f32p, i32, i32, i32, f32, i32p, i32p, i32p, f32p, i32p]
    L.mt_place_window.argtypes = [f32p, i32, i32, i32, f32p, u8p]
    L.mt_check.argtypes = [i32, i32, i32, f32, f32, i32, f32, f32, f32, f32]
    L.mt_check.restype = C.c_char_p
    return L


def packed_bands(L, fb):
    """(lo, hi) of every mel as the plan's packer (pack_bands) lays them out."""
    n_mels, bins = fb.shape
    fb = np.ascontiguousarray(fb, F32).reshape(-1)
    nnz, n_slots = C.c_int32(), C.c_int32()
    L.mt_pack_sizes(fb, n_mels, bins, C.byref(nnz), C.byref(n_slots))
    lo, hi, off = (np.zeros(n_mels, np.int32) for _ in range(3))
    w = np.zeros(max(nnz.value, 1), F32)
    slots = np.zeros(max(n_slots.value, 1) * 4, np.int32)
    L.mt_pack(fb, n_mels, bins, 0, 1.0, lo, hi, off, w, slots)
    return lo, hi


def cpu_tables(L, cfg: Cfg):
    """The handle's window [win] and table [M x bins], as fa_mel_create_ex builds them."""
    w = np.zeros(cfg.win, F32)
    fb = np.zeros((cfg.n_mels, cfg.n_fft // 2 + 1), F32)
    L.mt_tables(cfg.sample_rate, cfg.n_mels, cfg.n_fft, cfg.win, int(cfg.periodic), cfg.kind, cfg.filter_sr, cfg.f_min,
                cfg.f_max, w, fb.reshape(-1))
    return w, fb


def with_(cfg: Cfg, **kw) -> Cfg:
    return replace(cfg, **kw)
