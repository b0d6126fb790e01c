"""The C ABI of the LS-EEND feature streams (``include/fluidaudio_b200_lseend.h``, ``fluidaudio_b200/csrc/lseend/``) keeps
the library's ABI rules, on the CPU: the header is plain C11; every function it declares is exported and bound in
``_lib.LSEEND_SYMBOLS``; each status-returning entry point refused before any CUDA call (a null handle or a null required
pointer) returns its status and leaves fa_last_error() text of its own; ``fa_lseend_stream_chunks`` refuses with -1 and
text; and every status-returning entry point is a body that returns through the one guard (``csrc/c_abi.h``)."""
import ctypes as C
import os
import re
import subprocess

import pytest

from fluidaudio_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "fluidaudio_b200_lseend.h")
FAMILY = os.path.join(ROOT, "fluidaudio_b200", "csrc", "lseend")

N = None
i32, i64, sz = C.c_int32, C.c_int64, C.c_size_t

# entry point -> (status, arguments it refuses before touching the device)
REFUSED = {
    "fa_lseend_stream_resolve": (1, [N, N]),
    "fa_lseend_stream_create": (1, [N, N]),
    "fa_lseend_stream_open": (1, [N, N]),
    "fa_lseend_stream_close": (1, [N, i32(0)]),
    "fa_lseend_stream_push": (1, [N, i32(0), N, N, N, N, N, sz(0), N, sz(0), N, sz(0), N]),
    "fa_lseend_stream_push_device": (1, [N, i32(0), N, N, N, N, N, sz(0), N, sz(0), N, sz(0), N]),
    "fa_lseend_stream_snapshot": (1, [N, i32(0), N]),
    "fa_lseend_stream_rollback": (1, [N, i32(0), N]),
    "fa_lseend_stream_reset": (1, [N, i32(0), N]),
    "fa_lseend_stream_session_state": (1, [N, i32(0), N, N, N, N]),
}
COUNTS = {"fa_lseend_stream_chunks": [N, i32(0), i64(0), i32(0)]}
VOID = {"fa_lseend_stream_destroy"}   # NULL is a no-op


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
    L.fa_lseend_stream_chunks.restype = i64
    return L


def test_every_declared_entry_point_is_covered_exported_and_bound(lib):
    declared = _declared()
    assert declared == set(REFUSED) | set(COUNTS) | VOID == set(_lib.LSEEND_SYMBOLS)
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    assert declared <= exported


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "lseend_header.c"
    src.write_text('#include "fluidaudio_b200_lseend.h"\nint main(void) { return (int)sizeof(fa_lseend_stream_config); }\n')
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I",
                           os.path.join(ROOT, "include"), str(src)])


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


def test_a_refused_count_reports_its_own_failure(lib):
    sentinel = _sentinel(lib)
    assert lib.fa_lseend_stream_chunks(*COUNTS["fa_lseend_stream_chunks"]) == -1
    text = lib.fa_last_error()
    assert text and text != sentinel


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
