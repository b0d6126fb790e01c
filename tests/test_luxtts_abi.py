"""The C ABI of LuxTTS synthesis (``include/fluidaudio_b200_luxtts.h``, ``fluidaudio_b200/csrc/luxtts/``) keeps the
library's ABI rules, on the CPU: the header is plain C11; every function it declares is exported and bound in
``_lib.LUXTTS_SYMBOLS``; each status-returning entry point refused before any CUDA call returns its status and leaves
fa_last_error() text of its own; every status-returning entry point returns through the one guard and nothing catches;
every kernel launch goes through the counting helpers and no CUDA buffer or stream is made outside their owners; and
the documented constants are the kernels'."""
import ctypes as C
import math
import os
import re
import subprocess

import pytest

from fluidaudio_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "fluidaudio_b200_luxtts.h")
FAMILY = os.path.join(ROOT, "fluidaudio_b200", "csrc", "luxtts")

N = None
i32, i64, sz = C.c_int32, C.c_int64, C.c_size_t

# entry point -> (status, arguments it refuses before touching the device)
REFUSED = {
    "fa_luxtts_plan": (1, [i64(-1), i32(1), i32(1), C.c_float(1.0), C.byref(_lib.LuxTtsPlanInfo())]),
    "fa_luxtts_create": (1, [N]),
    "fa_luxtts_begin": (1, [N, i32(1)] + [N] * 11),
    "fa_luxtts_begin_device": (1, [N, i32(1)] + [N] * 11),
    "fa_luxtts_text_condition": (1, [N, i32(0), N, N, i64(100), i64(100), N]),
    "fa_luxtts_text_condition_device": (1, [N, i32(0), N, N, i64(100), i64(100), N]),
    "fa_luxtts_model_inputs": (1, [N, i32(0), N, N, N]),
    "fa_luxtts_model_inputs_device": (1, [N, i32(0), N, N, N]),
    "fa_luxtts_advance": (1, [N, i32(0), N, N, i64(100), i64(100)]),
    "fa_luxtts_advance_device": (1, [N, i32(0), N, N, i64(100), i64(100)]),
    "fa_luxtts_vocoder_input": (1, [N, i32(0), N, i32(282), N]),
    "fa_luxtts_vocoder_input_device": (1, [N, i32(0), N, i32(282), N]),
    "fa_luxtts_finish": (1, [N, i32(0), N, N, i64(0), i64(0), N, sz(0), N, N]),
    "fa_luxtts_finish_device": (1, [N, i32(0), N, N, i64(0), i64(0), N, sz(0), N, N]),
    "fa_luxtts_close": (1, [N, i32(0)]),
    "fa_luxtts_request_state": (1, [N, i32(0), N, N]),
}
VOID = {"fa_luxtts_destroy"}   # NULL is a no-op


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
    assert declared == set(REFUSED) | VOID == set(_lib.LUXTTS_SYMBOLS)
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    assert declared <= exported


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "luxtts_header.c"
    src.write_text('#include "fluidaudio_b200_luxtts.h"\n'
                   'int main(void) { fa_luxtts_plan_info p; fa_luxtts *h = 0; (void)h;\n'
                   '  (void)fa_luxtts_plan(1000, 1, 1, 1.0f, &p);\n'
                   '  return FA_LUXTTS_FEAT_DIM + FA_LUXTTS_MAX_FRAMES + FA_LUXTTS_MAX_TOKENS + FA_LUXTTS_MAX_PROMPT\n'
                   '    + FA_LUXTTS_NUM_STEPS + FA_LUXTTS_HOP_48K + FA_LUXTTS_SAMPLE_RATE + FA_LUXTTS_DEGENERATE_DURATION; }\n')
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I",
                           os.path.join(ROOT, "include"), str(src)])


def test_the_documented_constants_are_the_kernels():
    text = open(HEADER).read()
    core = open(os.path.join(FAMILY, "luxtts_core.cuh")).read()
    kernels = open(os.path.join(FAMILY, "luxtts_kernels.cu")).read()
    for name, value in (("FEAT_DIM", 100), ("MAX_FRAMES", 1024), ("MAX_TOKENS", 256), ("MAX_PROMPT", 120000),
                        ("NUM_STEPS", 4), ("HOP_48K", 512), ("SAMPLE_RATE", 48000)):
        assert re.search(rf"#define FA_LUXTTS_{name} {value}\b", text), name
    for decl in ("kFeat = 100;", "kMaxFrames = 1024;", "kMaxTokens = 256;", "kMaxPrompt = 120000;", "kSteps = 4;",
                 "kHop48k = 512;", "kBucketSmall = 282, kBucketLarge = 555;", "kRmsLanes = 256;",
                 "kGamma = 0x9E3779B97F4A7C15ull;", "kSeedZero = 0xDEADBEEFCAFEBABEull;"):
        assert decl in core, decl
    assert "kFeatScale = 0.1f, kTargetRms = 0.1f;" in kernels
    reasons = re.findall(r"FA_LUXTTS_([A-Z_]+) = (\d+)", text)
    assert [int(v) for _, v in reasons] == list(range(12))
    # invScale and logFloor as the header states them, in float32
    import numpy as np
    assert np.float32(1) / np.float32(0.1) == np.float32(10.0)
    assert np.float32(math.log(np.float32(1e-7))) == np.float32(-16.118095)


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
        for m in re.finditer(r"\b(?:FA_API\s+fa_status|FA_LUXTTS_API)\s+(\w+)\s*\(", code):
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
    # every exported definition of the family is a guarded status entry point or the void destroy
    exported = set()
    for name in sorted(os.listdir(FAMILY)):
        exported |= set(re.findall(r"\bFA_(?:LUXTTS_)?API\s+(?:\w+\s+)*?(fa_\w+)\s*\(", _code(os.path.join(FAMILY, name))))
    assert exported == set(REFUSED) | VOID


def test_every_launch_goes_through_the_counting_helpers():
    offenders = []
    for name in sorted(os.listdir(FAMILY)):
        code = re.sub(r"/\*.*?\*/|//[^\n]*", " ", open(os.path.join(FAMILY, name), encoding="utf-8").read(), flags=re.S)
        offenders += [f"{name}: {t}" for t in ("<<<", "cudaLaunchCooperativeKernel", "cudaLaunchKernel") if t in code]
        offenders += [f"{name}: {m}" for m in re.findall(r"\b(cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*)\s*\(", code)]
    assert not offenders
    assert "launch(" in open(os.path.join(FAMILY, "luxtts_kernels.cu")).read()
