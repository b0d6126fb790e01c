"""The C ABI of streaming speaker tracking (``include/fluidaudio_b200_online_diar.h``,
``fluidaudio_b200/csrc/online_diar/``) keeps the
library's ABI rules, on the CPU: the header is plain C11; every function it declares is exported and bound in
``_lib.ONLINE_DIAR_SYMBOLS``; each status-returning entry point refused before any CUDA call returns its status and leaves
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
HEADER = os.path.join(ROOT, "include", "fluidaudio_b200_online_diar.h")
FAMILY = os.path.join(ROOT, "fluidaudio_b200", "csrc", "online_diar")

N = None
i32, i64, sz, vp = C.c_int32, C.c_int64, C.c_size_t, C.c_void_p
_off = np.array([0, 1], np.int64)
_bad_off = np.array([1, 2], np.int64)
_cfg = _lib.OnlineDiarConfig(0.7, 1.0, 2.0, 0.5, -1, 10.0, 10.0, 0.0)
_bad_cfg = _lib.OnlineDiarConfig(0.7, 1.0, 2.0, 0.5, -1, 10.0, 10.0, 10.0)   # a step of 0

# entry point -> (status, arguments it refuses before touching the device)
REFUSED = {
    "fa_od_resolve": (1, [C.byref(_bad_cfg), C.byref(_lib.OnlineDiarResolved())]),
    "fa_od_chunk_inputs": (1, [N, vp(_bad_off.ctypes.data), i32(1), i64(160000), N, N]),
    "fa_od_chunk_inputs_device": (1, [N, vp(_off.ctypes.data), i32(1), i64(0), N, N]),
    "fa_od_enrollment_inputs": (1, [N, vp(_off.ctypes.data), i32(1), i32(0), N, N]),
    "fa_od_enrollment_inputs_device": (1, [N, vp(_off.ctypes.data), i32(-1), i32(589), N, N]),
    "fa_od_create": (1, [i32(589), N]),
    "fa_od_open": (1, [N, N]),
    "fa_od_close": (1, [N, i32(0)]),
    "fa_od_embedding_inputs": (1, [N, i32(0), N, N, C.byref(_cfg), N, N]),
    "fa_od_embedding_inputs_device": (1, [N, i32(0), N, N, N, N, N]),
    "fa_od_advance": (1, [N, i32(0), N, N, N, C.byref(_cfg), N, N, N, N]),
    "fa_od_advance_device": (1, [N, i32(0), N, N, N, N, N, N, N, N]),
    "fa_od_query": (1, [N, i32(0), i32(0), N, N]),
    "fa_od_query_device": (1, [N, i32(0), i32(0), N, N]),
    "fa_od_speaker_count": (1, [N, i32(0), N, N]),
    "fa_od_read": (1, [N, i32(0), N, N, N]),
    "fa_od_initialize": (1, [N, i32(0), i32(0), N, N, N, i32(0), i32(1)]),
    "fa_od_remove": (1, [N, i32(0), i32(0), i64(1), i32(1), N]),
    "fa_od_merge": (1, [N, i32(0), i32(0), i64(1), i32(0), i64(2), i32(1), N]),
    "fa_od_set_permanent": (1, [N, i32(0), i32(0), i64(1), i32(1), N]),
    "fa_od_reset": (1, [N, i32(0), i32(0)]),
    "fa_od_upsert": (1, [N, i32(0), N, N, N]),
}
VOID = {"fa_od_default_config", "fa_od_destroy"}   # NULL is a no-op


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
    assert declared == set(REFUSED) | VOID == set(_lib.ONLINE_DIAR_SYMBOLS)
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    assert declared <= exported


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "od_header.c"
    src.write_text('#include "fluidaudio_b200_online_diar.h"\n'
                   'int main(void) { fa_od_config c; fa_od_resolved r; fa_od_speaker s; fa_od_default_config(&c);\n'
                   '  (void)s; (void)fa_od_resolve(&c, &r);\n'
                   '  return FA_OD_DIM + FA_OD_FIFO + FA_OD_CLASSES + FA_OD_LOCAL + FA_OD_MODEL_SAMPLES + FA_OD_MODE_SKIP; }\n')
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I",
                           os.path.join(ROOT, "include"), str(src)])


def test_the_documented_constants_are_the_kernels():
    text = open(HEADER).read()
    core = open(os.path.join(FAMILY, "online_diar_core.cuh")).read()
    for name, value in (("DIM", 256), ("FIFO", 50), ("CLASSES", 7), ("LOCAL", 3), ("MODEL_SAMPLES", 160000)):
        assert re.search(rf"#define FA_OD_{name} {value}\b", text)
    for name, value in (("kDim", 256), ("kFifo", 50), ("kClasses", 7), ("kLocal", 3), ("kModelSamples", 160000)):
        assert f"{name} = {value};" in core
    assert "sizeof(fa::od::SpeakerView) == sizeof(fa_od_speaker)" in open(os.path.join(FAMILY, "online_diar_abi.cu")).read()
    assert _lib.ONLINE_DIAR_SPEAKER.itemsize == 48


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
    assert "launch(" in open(os.path.join(FAMILY, "online_diar_kernels.cu")).read()
