"""The C ABI of offline Sortformer windows (``include/fluidaudio_b200_offline_sortformer.h``,
``fluidaudio_b200/csrc/offline_sortformer/``) keeps the library's ABI rules, on the CPU: the header is plain C11; every
function it declares is exported and bound in ``_lib.OFFLINE_SORTFORMER_SYMBOLS``; each entry point refused before any
CUDA call returns its status, leaves fa_last_error() text of its own and writes nothing; every entry point returns
through the one guard and nothing catches; every kernel launch goes through the counting helpers and no CUDA buffer or
stream is made outside their owners; and the documented constants are the kernels'."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from fluidaudio_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "fluidaudio_b200_offline_sortformer.h")
FAMILY = os.path.join(ROOT, "fluidaudio_b200", "csrc", "offline_sortformer")

N = None
i32, i64 = C.c_int32, C.c_int64


def P(a):
    return C.c_void_p(a.ctypes.data)


# entry point -> (status, arguments it refuses before touching the device)
REFUSED = {
    "fa_offline_sortformer_plan": (1, [i32(100), i32(1), N, N, N]),
    "fa_offline_sortformer_model_inputs": (1, [i32(100), i32(-1), N, N, N, i64(0), N, N]),
    "fa_offline_sortformer_model_inputs_device": (1, [i32(100), i32(1), N, N, N, i64(0), N, N]),
    "fa_offline_sortformer_stitch": (1, [i32(100), i32(1), N, N, N, N]),
    "fa_offline_sortformer_stitch_device": (1, [i32(100), i32(-3), N, N, N, N]),
}

def _declared():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return set(re.findall(r"\b(fa_[a-z0-9_]+)\s*\(", text))


def _code(path):
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", open(path, encoding="utf-8").read(), flags=re.S)
    return re.sub(r'"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', '""', text)


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    L = C.CDLL(_lib.LIB_PATH)   # its own function objects: every argument below carries its C type
    L.fa_last_error.restype = C.c_char_p
    return L


def test_every_declared_entry_point_is_covered_exported_and_bound(lib):
    declared = _declared()
    assert declared == set(REFUSED) == set(_lib.OFFLINE_SORTFORMER_SYMBOLS)
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    assert declared <= exported


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "offline_sortformer_header.c"
    src.write_text('#include "fluidaudio_b200_offline_sortformer.h"\n'
                   'int main(void) { int64_t n = 5, w, r;\n'
                   '  (void)fa_offline_sortformer_plan(100, 1, &n, &w, &r);\n'
                   '  return FA_OFFLINE_SORTFORMER_WINDOW_OUT + FA_OFFLINE_SORTFORMER_SUBSAMPLING\n'
                   '    + FA_OFFLINE_SORTFORMER_WINDOW_MEL + FA_OFFLINE_SORTFORMER_SPEAKERS + FA_OFFLINE_SORTFORMER_MELS\n'
                   '    + FA_OFFLINE_SORTFORMER_DEFAULT_OVERLAP; }\n')
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I",
                           os.path.join(ROOT, "include"), str(src)])


def test_the_documented_constants_are_the_kernels():
    text = open(HEADER).read()
    core = open(os.path.join(FAMILY, "offline_sortformer_core.cuh")).read()
    for name, value in (("WINDOW_OUT", 384), ("SUBSAMPLING", 8), ("WINDOW_MEL", 3072), ("SPEAKERS", 4), ("MELS", 128),
                        ("DEFAULT_OVERLAP", 100)):
        assert re.search(rf"#define FA_OFFLINE_SORTFORMER_{name} {value}\b", text), name
    for decl in ("kWindowOut = 384;", "kSubsampling = 8;", "kWindowMel = kWindowOut * kSubsampling;",
                 "kSpeakers = 4;", "kMels = 128;", "kPerms = 24;", "kDefaultOverlap = 100;"):
        assert decl in core, decl
    from fluidaudio_b200 import offline_sortformer as OS
    assert (OS.WINDOW_OUT, OS.SUBSAMPLING, OS.WINDOW_MEL, OS.SPEAKERS, OS.MELS) == (384, 8, 3072, 4, 128)
    # the kernels use the rounded intrinsics: NVFLAGS leaves FMA contraction on
    assert "__fmul_rn" in core and "__fadd_rn" in core


def _sentinel(L):
    """a refused call of the main header that sets its own text"""
    fmt = _lib.AudioFormat(0.0, 16000.0, 1, 0, 0, 0)
    count = C.c_int64()
    assert L.fa_audio_resample(N, i64(10), C.byref(fmt), N, i64(0), C.byref(count)) == 1
    return L.fa_last_error()


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_a_refused_call_reports_its_own_failure(lib, name):
    status, args = REFUSED[name]
    sentinel = _sentinel(lib)
    assert getattr(lib, name)(*args) == status
    text = lib.fa_last_error()
    assert text and text != sentinel, f"{name} left {text!r}"


def test_every_status_entry_point_returns_through_the_guard():
    guarded, offenders = set(), []
    for name in sorted(os.listdir(FAMILY)):
        code = _code(os.path.join(FAMILY, name))
        assert not re.search(r"\bcatch\s*\(", code), f"{name} catches: only the guard maps exceptions"
        for m in re.finditer(r"\b(?:FA_API\s+fa_status|FA_OFFLINE_SORTFORMER_API)\s+(\w+)\s*\(", code):
            i = code.index("{", m.end())
            depth, j, statements = 1, i + 1, 0
            while depth:
                c = code[j]
                depth += {"{": 1, "(": 1, "[": 1, "}": -1, ")": -1, "]": -1}.get(c, 0)
                statements += c == ";" and depth == 1
                j += 1
            body = " ".join(code[i + 1:j - 1].split())
            if statements == 1 and re.match(r"return (fa::)?guard\(__func__, ", body):
                guarded.add(m.group(1))
            else:
                offenders.append(f"{name}: {m.group(1)}")
    assert not offenders, offenders
    assert guarded == set(REFUSED)
    exported = set()
    for name in sorted(os.listdir(FAMILY)):
        exported |= set(re.findall(r"\bFA_(?:OFFLINE_SORTFORMER_)?API\s+(?:\w+\s+)*?(fa_\w+)\s*\(", _code(os.path.join(FAMILY, name))))
    assert exported == set(REFUSED)


def test_every_launch_goes_through_the_counting_helpers():
    offenders = []
    for name in sorted(os.listdir(FAMILY)):
        code = re.sub(r"/\*.*?\*/|//[^\n]*", " ", open(os.path.join(FAMILY, name), encoding="utf-8").read(), flags=re.S)
        offenders += [f"{name}: {t}" for t in ("<<<", "cudaLaunchCooperativeKernel", "cudaLaunchKernel") if t in code]
        offenders += [f"{name}: {m}" for m in re.findall(r"\b(cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*)\s*\(", code)]
    assert not offenders
    assert "launch(" in open(os.path.join(FAMILY, "offline_sortformer_kernels.cu")).read()


# ------------------------------------------------------------------------------------------------ refusals write nothing
def _model_inputs(L, frames, offsets=None, capacity=None, device=False, mel=True):
    frames = np.asarray(frames, np.int64)
    offsets = np.concatenate([[0], np.cumsum(np.maximum(frames, 0) * 128)])[:-1].astype(np.int64) \
        if offsets is None else np.asarray(offsets, np.int64)
    m = np.zeros(max(int(np.minimum(np.maximum(frames, 0), 8192).sum()) * 128, 1), np.float32)
    W = 8 if capacity is None else capacity
    out, ml = np.full(max(W, 1) * 128 * 3072, 7, np.float32), np.full(max(W, 1), -9, np.int32)
    fn = L.fa_offline_sortformer_model_inputs_device if device else L.fa_offline_sortformer_model_inputs
    st = fn(i32(100), i32(frames.size), P(m) if mel else N, P(offsets), P(frames), i64(W), P(out), P(ml))
    return st, bool((out == 7).all() and (ml == -9).all())


@pytest.mark.parametrize("device", [False, True])
def test_model_inputs_refusals_write_nothing(lib, device):
    for kw, status in ((dict(frames=[3, -1]), 1), (dict(frames=[3, (1 << 40) + 1]), 1),
                       (dict(frames=[3, 4], offsets=[0, -128]), 1), (dict(frames=[3], capacity=-1), 1),
                       (dict(frames=[3], mel=False), 1), (dict(frames=[5344, 3073], capacity=4), 3),
                       (dict(frames=[3072], capacity=1), 3), (dict(frames=[3, 4], offsets=[0, (1 << 62) - 100]), 1)):
        st, untouched = _model_inputs(lib, device=device, **kw)
        assert st == status and untouched, kw
        assert lib.fa_last_error()
    assert b"window_capacity" in lib.fa_last_error() or b"offsets" in lib.fa_last_error()
    assert lib.fa_offline_sortformer_model_inputs(i32(100), i32(0), N, N, N, i64(0), N, N) == 0   # nothing to do
    z = np.zeros(2, np.int64)
    assert lib.fa_offline_sortformer_model_inputs(i32(100), i32(2), N, P(z), P(z), i64(0), N, N) == 0   # no window


@pytest.mark.parametrize("device", [False, True])
def test_stitch_refusals_write_nothing(lib, device):
    fn = lib.fa_offline_sortformer_stitch_device if device else lib.fa_offline_sortformer_stitch
    preds = np.zeros(3 * 384 * 4, np.float32)
    for frames, p in (([3, -1], preds), ([3, 1 << 41], preds), ([3], None)):
        n = np.asarray(frames, np.int64)
        out, maps = np.full(64, 7, np.float32), np.full(64, -9, np.int32)
        assert fn(i32(100), i32(n.size), P(n), N if p is None else P(p), P(out), P(maps)) == 1
        assert (out == 7).all() and (maps == -9).all() and lib.fa_last_error()
    assert fn(i32(100), i32(-1), N, N, N, N) == 1 and b"count" in lib.fa_last_error()
    assert fn(i32(100), i32(0), N, N, N, N) == 0


def test_plan_refusals_write_nothing(lib):
    n = np.array([3, -2], np.int64)
    w, r = np.full(2, -9, np.int64), np.full(2, -9, np.int64)
    assert lib.fa_offline_sortformer_plan(i32(7), i32(2), P(n), P(w), P(r)) == 1
    assert (w == -9).all() and (r == -9).all()
    assert lib.fa_offline_sortformer_plan(i32(7), i32(-1), N, N, N) == 1
    assert lib.fa_offline_sortformer_plan(i32(7), i32(0), N, N, N) == 0
