"""The C ABI of CTC decoding (``include/fluidaudio_b200_ctc_decode.h``, ``fluidaudio_b200/csrc/ctc_decode/``) keeps the
library's ABI rules, on the CPU: the header is plain C11; every function it declares is exported and bound in
``_lib.CTC_DECODE_SYMBOLS``; each status-returning entry point refused before any CUDA call returns its status and
leaves fa_last_error() text of its own; every status-returning entry point returns through the one guard; every kernel
launch goes through the counting helpers; and the documented limits are the kernels' constants."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from fluidaudio_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "fluidaudio_b200_ctc_decode.h")
FAMILY = os.path.join(ROOT, "fluidaudio_b200", "csrc", "ctc_decode")

N = None
i32, i64, f32, sz, vp = C.c_int32, C.c_int64, C.c_float, C.c_size_t, C.c_void_p
_off = np.array([0, 1], np.int64)
_bad_off = np.array([1, 2], np.int64)

# entry point -> (status, arguments it refuses before touching the device)
REFUSED = {
    "fa_ctc_lm_create": (1, [i32(-1), N, N, N, N, N, i64(0), N, N, N, N]),
    "fa_ctc_decoder_create": (1, [i32(0), i32(0), N, N, N]),
    "fa_ctc_beam_search": (1, [N, N, N, N, i32(0), N, N, N, N, sz(0), N]),
    "fa_ctc_beam_search_device": (1, [N, N, N, N, i32(-1), N, N, N, N, sz(0), N]),
    "fa_ctc_greedy": (1, [N, vp(_bad_off.ctypes.data), i32(1), i32(5), i32(4), N, N, sz(0), C.byref(C.c_int64())]),
    "fa_ctc_greedy_device": (1, [N, vp(_off.ctypes.data), i32(1), i32(0), i32(4), N, N, sz(0), C.byref(C.c_int64())]),
}
VOID = {"fa_ctc_beam_default_config", "fa_ctc_lm_destroy", "fa_ctc_decoder_destroy"}   # NULL is a no-op


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
    assert declared == set(REFUSED) | VOID == set(_lib.CTC_DECODE_SYMBOLS)
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    assert declared <= exported


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "ctc_decode_header.c"
    src.write_text('#include "fluidaudio_b200_ctc_decode.h"\n'
                   'int main(void) { fa_ctc_beam_config c; fa_ctc_beam_default_config(&c);\n'
                   '  return c.beam_width + FA_CTC_DECODE_MAX_BEAM_WIDTH + FA_CTC_DECODE_MAX_TOKEN_CANDIDATES; }\n')
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I",
                           os.path.join(ROOT, "include"), str(src)])


def test_the_documented_limits_are_the_kernels():
    text = open(HEADER).read()
    core = open(os.path.join(FAMILY, "ctc_decode_core.cuh")).read()
    for name, value in (("BEAM_WIDTH", 128), ("TOKEN_CANDIDATES", 64)):
        assert f"#define FA_CTC_DECODE_MAX_{name} {value}" in text
    assert "kMaxBeamWidth = 128;" in core and "kMaxTokenCandidates = 64;" in core
    # a frame's slots index 14 bits of an order key: 128 x (64 + 1) < 2^14
    assert 128 * 65 < 1 << 14 and "key & 0x3fff" in core


def test_default_config_is_the_reference_defaults(lib):
    cfg = _lib.CtcBeamConfig()
    lib.fa_ctc_beam_default_config(C.byref(cfg))
    assert (cfg.beam_width, cfg.token_candidates, cfg.lm_weight, cfg.word_bonus) == (100, 40, np.float32(0.3), 0.0)


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


def _lm_call(lib, words, has, lp, ctx, wd, blp):
    data = [w.encode() for w in words]
    buf = np.frombuffer(b"".join(data) + b"\0", np.uint8).copy()
    off = np.concatenate([[0], np.cumsum([len(d) for d in data])]).astype(np.int64)
    has, lp = np.array(has, np.int32), np.array(lp, np.float32)
    bo = np.zeros(len(words), np.float32)
    ctx, wd, blp = np.array(ctx, np.int32), np.array(wd, np.int32), np.array(blp, np.float32)
    out = C.c_void_p(7)
    st = lib.fa_ctc_lm_create(i32(len(words)), vp(buf.ctypes.data), vp(off.ctypes.data), vp(has.ctypes.data),
                              vp(lp.ctypes.data), vp(bo.ctypes.data), i64(len(ctx)), vp(ctx.ctypes.data),
                              vp(wd.ctypes.data), vp(blp.ctypes.data), C.byref(out))
    return st, out.value, lib.fa_last_error()


@pytest.mark.parametrize("case,text", [
    ((["a", "b", "a"], [1, 1, 1], [-1, -1, -1], [], [], []), b"word 2 repeats"),
    ((["a", "b"], [1, 1], [-1, -1], [0, 0], [1, 1], [-1, -2]), b"bigram 1 repeats"),
    ((["a", "b"], [1, 1], [-1, -1], [0], [2], [-1]), b"outside [0, 2)"),
    ((["a", "b"], [1, 1], [-1, float("inf")], [], [], []), b"non-finite unigram"),
    ((["a", "b"], [1, 0], [-1, 0], [1], [0], [float("nan")]), b"non-finite log-prob"),
])
def test_bad_language_models_are_refused(lib, case, text):
    _sentinel(lib)
    st, out, err = _lm_call(lib, *case)
    assert st == 1 and out is None and text in err, err


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
    assert "launch(" in open(os.path.join(FAMILY, "ctc_decode_kernels.cu")).read()
