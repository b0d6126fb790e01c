"""The C ABI of voice activity detection (``include/fluidaudio_b200_vad.h``, ``fluidaudio_b200/csrc/vad/``) keeps the
library's ABI rules, on the CPU: the header is plain C11; every function it declares is exported and bound in
``_lib.VAD_SYMBOLS``; each status-returning entry point refused before any CUDA call returns its status and leaves
fa_last_error() text of its own; every status-returning entry point returns through the one guard and nothing catches;
every kernel launch goes through the counting helpers and no CUDA buffer or stream is made outside their owners; and
the documented constants are the kernels'."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from fluidaudio_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "fluidaudio_b200_vad.h")
FAMILY = os.path.join(ROOT, "fluidaudio_b200", "csrc", "vad")

N = None
i32, i64, sz, vp = C.c_int32, C.c_int64, C.c_size_t, C.c_void_p
_off = np.array([0, 1], np.int64)
_bad_off = np.array([1, 2], np.int64)
_cfg = _lib.VadConfig(0.85, 0.15, 0.75, 14.0, 0.1, 0.3, 0, 0.0, 0.15, 0.098, 1)
_bad_cfg = _lib.VadConfig(0.85, -1.0, 0.75, 14.0, 0.1, 0.3, 0, 0.0, 0.15, 0.098, 1)

# entry point -> (status, arguments it refuses before touching the device)
REFUSED = {
    "fa_vad_resolve": (1, [C.byref(_bad_cfg), C.byref(_lib.VadResolved())]),
    "fa_vad_stream_create": (1, [N]),
    "fa_vad_stream_open": (1, [N, N]),
    "fa_vad_stream_close": (1, [N, i32(0)]),
    "fa_vad_stream_model_inputs": (1, [N, i32(0), N, N, N, N, N, N]),
    "fa_vad_stream_model_inputs_device": (1, [N, i32(1), N, N, N, N, N, N]),
    "fa_vad_stream_advance": (1, [N, i32(0), N, N, N, N, C.byref(_cfg), N]),
    "fa_vad_stream_advance_device": (1, [N, i32(0), N, N, N, N, N, N]),
    "fa_vad_stream_session_state": (1, [N, i32(0), N, N, N, N]),
    "fa_vad_segment": (1, [N, vp(_bad_off.ctypes.data), i32(1), N, C.byref(_cfg), N, N, sz(0),
                           C.byref(C.c_int64())]),
    "fa_vad_segment_device": (1, [N, vp(_off.ctypes.data), i32(1), N, C.byref(_bad_cfg), N, N, sz(0),
                                  C.byref(C.c_int64())]),
    "fa_fsmn_vad_decide": (1, [N, vp(_off.ctypes.data), i32(-1), N, N, sz(0), C.byref(C.c_int64())]),
    "fa_fsmn_vad_decide_device": (1, [N, vp(_off.ctypes.data), i32(1), N, N, sz(0), C.byref(C.c_int64())]),
}
VOID = {"fa_vad_default_config", "fa_vad_stream_destroy"}   # NULL is a no-op


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
    assert declared == set(REFUSED) | VOID == set(_lib.VAD_SYMBOLS)
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    assert declared <= exported


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "vad_header.c"
    src.write_text('#include "fluidaudio_b200_vad.h"\n'
                   'int main(void) { fa_vad_config c; fa_vad_resolved r; fa_vad_default_config(&c);\n'
                   '  fa_vad_stream_session_info i; (void)i; (void)fa_vad_resolve(&c, &r);\n'
                   '  return FA_VAD_CHUNK + FA_VAD_CONTEXT + FA_VAD_STATE + FA_VAD_MODEL_INPUT; }\n')
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I",
                           os.path.join(ROOT, "include"), str(src)])


def test_the_documented_constants_are_the_kernels():
    text = open(HEADER).read()
    core = open(os.path.join(FAMILY, "vad_core.cuh")).read()
    for name, value in (("CHUNK", 4096), ("CONTEXT", 64), ("STATE", 128), ("MODEL_INPUT", 4160)):
        assert f"#define FA_VAD_{name} {value}" in text
    assert "kChunk = 4096;" in core and "kContext = 64;" in core and "kState = 128;" in core
    assert "kModelInput = kContext + kChunk;" in core and 64 + 4096 == 4160


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
        offenders += [f"{name}: {m}" for m in re.findall(r"\b(cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*)\s*\(", code)]
    assert not offenders
    assert "launch(" in open(os.path.join(FAMILY, "vad_kernels.cu")).read()
