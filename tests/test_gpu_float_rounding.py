"""fa_float.cuh's f_exp / f_log / f_log1p on the H100, on every float32 input (tests/device/fa_float_probe.cu, built by
__graft_entry__.build()), against the reference of tests/test_float_rounding.py: glibc's float64 result rounded to
float32, with mpmath's correctly rounded value wherever that result lies within 3 float64 ulps of a rounding boundary.

Each function's 2^32 inputs go in 16 chunks of 2^28: the host computes a chunk's reference, the probe uploads it and
compares on the device (1 GiB of reference, nothing else resident).  The old policy, (float)f((double)x) with CUDA's
float64 libm, is evaluated on the fragile inputs and its disagreements with glibc and with the correct rounding are
printed: a measured finding (DESIGN §4.7), not an assertion.
"""
import ctypes
import os

import numpy as np
import pytest

import float_exact as FE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = 1 << 28
CAP = 64

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def probe(gpu_lib):
    path = os.path.join(ROOT, "tests", "device", "libfa_float_probe.so")
    assert os.path.exists(path), "tests/device/libfa_float_probe.so is missing: run __graft_entry__.build()"
    L = ctypes.CDLL(path)
    vp, u64, i32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_int
    L.fa_float_probe.argtypes = [i32, i32, u64, u64, vp, vp, vp, vp, i32, vp]
    L.fa_float_probe.restype = i32
    return L


@pytest.fixture(scope="module")
def reference(tmp_path_factory):
    L = FE.reference_library(tmp_path_factory.mktemp("float_reference"))
    return L, [FE.fragile_table(L, fn) for fn in range(3)]


def _hex(b):
    return float(np.uint32(b).view(np.float32)).hex()


@pytest.mark.parametrize("fn", [FE.EXP, FE.LOG, FE.LOG1P], ids=FE.NAMES)
def test_device_helpers_are_correctly_rounded_on_every_input(probe, reference, fn):
    L, tables = reference
    fin, fval = tables[fn]
    ref = np.empty(CHUNK, np.uint32)
    bad = np.zeros((CAP, 3), np.uint32)
    total, report = 0, []
    for start in range(0, 1 << 32, CHUNK):
        L.fr_reference(fn, start, CHUNK, None, fin.ctypes.data, fval.ctypes.data, len(fin), ref.ctypes.data)
        n = ctypes.c_ulonglong()
        assert probe.fa_float_probe(fn, 0, start, CHUNK, None, ref.ctypes.data, None, bad.ctypes.data, CAP,
                                    ctypes.byref(n)) == 0
        total += n.value
        report += [f"{FE.NAMES[fn]}({_hex(x)}) = {_hex(g)}, expected {_hex(w)}" for x, g, w in bad[:min(n.value, CAP)]]
    assert total == 0, f"{total} mismatches over all 2^32 inputs:\n" + "\n".join(report[:CAP])


def test_old_policy_on_the_fragile_inputs(probe, reference):
    """(float)f((double)x) with CUDA's float64 exp / log / log1p on the fragile inputs, reported against glibc's
    (float)f((double)x) and against the correct rounding."""
    _, tables = reference
    lines = []
    for fn, (xs, vals) in enumerate(tables):
        out = np.zeros(len(xs), np.uint32)
        n = ctypes.c_ulonglong()
        assert probe.fa_float_probe(fn, 1, 0, len(xs), xs.ctypes.data, None, out.ctypes.data, None, 0,
                                    ctypes.byref(n)) == 0
        glibc = np.array([FE._f32(FE._libm(fn, x)) for x in xs.view(np.float32)], np.float32).view(np.uint32)
        vs_glibc, vs_correct = int((out != glibc).sum()), int((out != vals).sum())
        lines.append(f"{FE.NAMES[fn]}: {len(xs)} fragile inputs, CUDA's old policy differs from glibc's at {vs_glibc} "
                     f"and from the correct rounding at {vs_correct} (glibc: {int((glibc != vals).sum())})")
        lines += [f"  {FE.NAMES[fn]}({_hex(x)}): cuda {_hex(o)}, glibc {_hex(g)}, correct {_hex(v)}"
                  for x, o, g, v in zip(xs, out, glibc, vals) if o != g or o != v]
    print("\n".join(lines))
    # the library's own helpers on the same inputs are the correctly rounded values
    for fn, (xs, vals) in enumerate(tables):
        n = ctypes.c_ulonglong()
        assert probe.fa_float_probe(fn, 0, 0, len(xs), xs.ctypes.data, vals.ctypes.data, None, None, 0,
                                    ctypes.byref(n)) == 0 and n.value == 0
