"""Correctly rounded float32 exp, log and log1p for the Python restatements.

Each function returns the float32 nearest the exact function of its float32 argument, the definition
``fluidaudio_b200/csrc/fa_float.cuh`` and ``oracle/oracle_float.h`` implement (DESIGN §4.7).  It evaluates
``math.f(float64(x))`` and rounds once to float32; where that float64 result lies within 3 float64 ulps of a point at
which the float32 rounding changes, it resolves the input with mpmath at 300 bits instead, because a float64 result
that close can round to the wrong float32 (double rounding), and two libms that are each within 1 ulp can disagree.
"""
import math
import struct

import mpmath
import numpy as np

F = np.float32
WINDOW = 3
EXP, LOG, LOG1P = 0, 1, 2
NAMES = ("exp", "log", "log1p")
_MATH = (math.exp, math.log, math.log1p)
_FLT_MAX = float(np.finfo(np.float32).max)
_OVERFLOW = 2.0 ** 128 - 2.0 ** 103   # float32 rounding reaches inf from here up


def _step(a, n):
    """|a| moved n float64 ulps away from zero (never below zero)."""
    b = struct.unpack("<q", struct.pack("<d", a))[0]
    return struct.unpack("<d", struct.pack("<q", max(0, b + n)))[0]


def _f32(d):
    """float64 -> float32, round to nearest even, overflowing to inf as a C cast does."""
    return F(math.copysign(math.inf, d)) if abs(d) >= _OVERFLOW else F(d)


def fragile(d):
    """Whether float32 rounding of the float64 d changes within WINDOW float64 ulps of it."""
    if not math.isfinite(d):
        return False
    a = abs(d)
    return _f32(_step(a, -WINDOW)) != _f32(_step(a, WINDOW))


def _libm(fn, x):
    x = float(x)
    if fn == LOG and x <= 0:
        return -math.inf if x == 0 else math.nan
    if fn == LOG1P and x <= -1:
        return -math.inf if x == -1 else math.nan
    if fn == EXP and x > 709:
        return math.inf
    try:
        return _MATH[fn](x)
    except ValueError:
        return math.nan


def correctly_rounded(fn, x):
    """The float32 nearest fn(x), for a finite float32 x where fn(x) is finite and not exactly a float32, by mpmath."""
    with mpmath.workprec(300):
        v = mpmath.mpf(float(F(x)))
        v = mpmath.exp(v) if fn == EXP else mpmath.log(v) if fn == LOG else mpmath.log(1 + v)
        # the float32 grid at |v|: 24 significant bits, never finer than the subnormal spacing 2^-149
        e = max(int(mpmath.floor(mpmath.log(abs(v), 2))) - 23, -149)
        q = mpmath.nint(mpmath.ldexp(v, -e))
        r = float(mpmath.ldexp(q, e))
    return _f32(r) if abs(r) <= _FLT_MAX else F(math.copysign(math.inf, r))


def f32(fn, x):
    """The correctly rounded float32 fn(x) for one float32 x."""
    d = _libm(fn, F(x))
    return correctly_rounded(fn, x) if fragile(d) else _f32(d)


def exp(x):
    return f32(EXP, x)


def log(x):
    return f32(LOG, x)


def log1p(x):
    return f32(LOG1P, x)


def vectorized(fn, a):
    """f32(fn, .) over a float32 array, same shape."""
    a = np.asarray(a, np.float32)
    return np.array([f32(fn, x) for x in a.ravel()], np.float32).reshape(a.shape)


# ---- the exhaustive reference: tests/emul/float_reference.cpp over all 2^32 inputs ----

def reference_library(out_dir):
    """Compiles tests/emul/float_reference.cpp into out_dir and returns it loaded, argument types set."""
    import ctypes
    import os
    import subprocess
    root = os.path.dirname(os.path.abspath(__file__))
    out = os.path.join(str(out_dir), "libfloat_reference.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-o", out,
                           os.path.join(root, "emul", "float_reference.cpp")])
    L = ctypes.CDLL(out)
    vp, i32, i64, u64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_uint64
    L.fr_scan.argtypes, L.fr_scan.restype = [i32, vp, i64], i64
    L.fr_reference.argtypes, L.fr_reference.restype = [i32, u64, u64, vp, vp, vp, i64, vp], None
    L.fr_check.argtypes, L.fr_check.restype = [i32, vp, vp, vp, i64, vp, i64], i64
    return L


def fragile_table(L, fn):
    """(inputs, values) as sorted uint32 bit arrays: every float32 input whose glibc float64 result is fragile, and its
    correctly rounded float32 by mpmath."""
    cap = 1 << 12
    xs = np.zeros(cap, np.uint32)
    n = L.fr_scan(fn, xs.ctypes.data, cap)
    assert n <= cap, n
    xs = xs[:n].copy()
    vals = np.array([correctly_rounded(fn, x) for x in xs.view(np.float32)], np.float32).view(np.uint32)
    return xs, vals
