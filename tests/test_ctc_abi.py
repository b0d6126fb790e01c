"""The C ABI of CTC keyword spotting (``include/fluidaudio_b200_ctc.h``, ``fluidaudio_b200/csrc/ctc/``) keeps the
library's ABI rules, on the CPU: the header is plain C11; every function it declares is exported and bound in
``_lib.CTC_SYMBOLS``; each status-returning entry point refused before any CUDA call returns its status and leaves
fa_last_error() text of its own; every status-returning entry point is a body that returns through the one guard
(``csrc/c_abi.h``); and every kernel launch under ``csrc/ctc/`` goes through the counting helpers of ``fa_common.cuh``."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from fluidaudio_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "fluidaudio_b200_ctc.h")
FAMILY = os.path.join(ROOT, "fluidaudio_b200", "csrc", "ctc")

N = None
i32, i64, f32, sz, vp = C.c_int32, C.c_int64, C.c_float, C.c_size_t, C.c_void_p
MAX_TOKENS = 127

# entry point -> (status, arguments it refuses before touching the device)
REFUSED = {
    "fa_ctc_log_softmax": (1, [N, i32(-1), i32(5), i32(0), f32(1), f32(0), i32(0), N]),
    "fa_ctc_log_softmax_device": (1, [N, i32(2), i32(5), i32(7), f32(1), f32(0), i32(0), N]),
    "fa_ctc_merge_chunks": (1, [N, N, i32(1), i32(5), i32(0), N, sz(0), N]),
    "fa_ctc_merge_chunks_device": (1, [N, N, i32(-1), i32(5), i32(0), N, sz(0), N]),
    "fa_ctc_spotter_create": (1, [i32(0), i32(0), i32(0), N, N, N]),
    "fa_ctc_spot": (1, [N, N, N, i32(0), N, N, N, N, sz(0)]),
    "fa_ctc_spot_device": (1, [N, N, N, i32(0), N, N, N, N, sz(0)]),
    "fa_ctc_spot_constrained": (1, [N, i32(-1), i32(5), i32(0), i32(0), N, N, N, N, N, N, N]),
    "fa_ctc_spot_constrained_device": (1, [N, i32(4), i32(0), i32(0), i32(0), N, N, N, N, N, N, N]),
}
VOID = {"fa_ctc_spotter_destroy"}   # NULL is a no-op


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
    assert declared == set(REFUSED) | VOID == set(_lib.CTC_SYMBOLS)
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    assert declared <= exported


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "ctc_header.c"
    src.write_text('#include "fluidaudio_b200_ctc.h"\n'
                   'int main(void) { return (int)sizeof(fa_ctc_detection) + FA_CTC_MAX_TERM_TOKENS; }\n')
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I",
                           os.path.join(ROOT, "include"), str(src)])


def test_the_documented_bound_is_the_kernels():
    text = open(HEADER).read()
    assert f"#define FA_CTC_MAX_TERM_TOKENS {MAX_TOKENS}" in text
    core = open(os.path.join(FAMILY, "ctc_core.cuh")).read()
    assert "kStatesPerLane = 8" in core and "kMaxTokens = (kMaxStates - 1) / 2" in core   # (32 x 8 - 1) / 2 = 127


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


def _offsets(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)


def test_more_tokens_than_supported_is_refused_with_its_own_text(lib):
    for n, st in ((MAX_TOKENS + 1, 8), (MAX_TOKENS + 40, 8)):
        tok = np.zeros(n + 2, np.int32)
        off = _offsets([2, n])
        out = C.c_void_p(7)
        _sentinel(lib)
        assert lib.fa_ctc_spotter_create(i32(5), i32(4), i32(2), vp(tok.ctypes.data), vp(off.ctypes.data), C.byref(out)) == st
        assert out.value is None
        assert b"term 1 has" in lib.fa_last_error()
        ss = np.zeros(2, np.int64)
        _sentinel(lib)
        assert lib.fa_ctc_spot_constrained(N, i32(0), i32(5), i32(4), i32(2), vp(tok.ctypes.data), vp(off.ctypes.data),
                                           vp(ss.ctypes.data), vp(ss.ctypes.data), vp(ss.ctypes.data), vp(ss.ctypes.data),
                                           vp(ss.ctypes.data)) == st
        assert b"query 1 has" in lib.fa_last_error()


@pytest.mark.parametrize("offsets", [[1, 2], [0, 3, 2], [0, -1]])
def test_bad_offsets_are_refused(lib, offsets):
    off = np.array(offsets, np.int64)
    tok = np.zeros(8, np.int32)
    out = C.c_void_p()
    assert lib.fa_ctc_spotter_create(i32(5), i32(4), i32(len(off) - 1), vp(tok.ctypes.data), vp(off.ctypes.data),
                                     C.byref(out)) == 1
    assert b"term_offsets" in lib.fa_last_error()
    rows = C.c_int32(-7)
    assert lib.fa_ctc_merge_chunks(vp(tok.ctypes.data), vp(off.ctypes.data), i32(len(off) - 1), i32(1), i32(0), vp(tok.ctypes.data),
                                   sz(8), C.byref(rows)) == 1
    assert rows.value == -7 and b"row_offsets" in lib.fa_last_error()


def test_negative_blank_with_a_bias_is_refused(lib):
    x = np.zeros(10, np.float32)
    assert lib.fa_ctc_log_softmax(vp(x.ctypes.data), i32(2), i32(5), i32(0), f32(1), f32(0.5), i32(-1), vp(x.ctypes.data)) == 1
    assert b"blank_id -1" in lib.fa_last_error()


def test_every_status_entry_point_returns_through_the_guard():
    guarded, offenders = set(), []
    for name in sorted(os.listdir(FAMILY)):
        code = _code(os.path.join(FAMILY, name))
        assert not re.search(r"\bcatch\s*\(", code), f"{name} catches: only the guard maps exceptions"
        for m in re.finditer(r"\bFA_API\s+fa_status\s+(\w+)\s*\(", code):
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


def test_every_launch_goes_through_the_counting_helpers():
    offenders = []
    for name in sorted(os.listdir(FAMILY)):
        code = re.sub(r"/\*.*?\*/|//[^\n]*", " ", open(os.path.join(FAMILY, name), encoding="utf-8").read(), flags=re.S)
        offenders += [f"{name}: {t}" for t in ("<<<", "cudaLaunchCooperativeKernel", "cudaLaunchKernel") if t in code]
    assert not offenders
    assert "launch(" in open(os.path.join(FAMILY, "ctc_kernels.cu")).read()
