"""The C ABI of StyleTTS2 synthesis glue (``include/fluidaudio_b200_styletts2.h``, ``fluidaudio_b200/csrc/styletts2/``)
keeps the library's ABI rules, on the CPU: the header is plain C11; every function it declares is exported and bound in
``_lib.STYLETTS2_SYMBOLS``; each entry point refused before any CUDA call returns its status, leaves fa_last_error()
text of its own and writes nothing but the reasons; every entry point returns through the one guard and nothing
catches; every kernel launch goes through the counting helpers and no CUDA buffer or stream is made outside their
owners; and the documented constants are the kernels'."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from fluidaudio_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "fluidaudio_b200_styletts2.h")
FAMILY = os.path.join(ROOT, "fluidaudio_b200", "csrc", "styletts2")

N = None
i32, i64 = C.c_int32, C.c_int64


def P(a):
    return C.c_void_p(a.ctypes.data)


ALIGN_NULLS = [N, N, i32(1), i64(1), i64(1), N, i32(1), i64(1), i64(1), N, i32(1), i64(1), i64(1), i64(1), N, N, N, N,
               N]

# entry point -> (status, arguments it refuses before touching the device)
REFUSED = {
    "fa_styletts2_plan": (1, [i32(5), N, N]),
    "fa_styletts2_sampler_inputs": (1, [i32(1), N, N, N, i32(57), N, N, N, N]),
    "fa_styletts2_sampler_inputs_device": (1, [i32(1), N, N, N, i32(57), N, N, N, N]),
    "fa_styletts2_style": (1, [i32(-1), N, N, N, N, N, N]),
    "fa_styletts2_style_device": (1, [i32(1), N, N, N, N, N, N]),
    "fa_styletts2_align": (1, [i32(1)] + ALIGN_NULLS),
    "fa_styletts2_align_device": (1, [i32(-2)] + ALIGN_NULLS),
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
    assert declared == set(REFUSED) == set(_lib.STYLETTS2_SYMBOLS)
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    assert declared <= exported


def test_header_is_plain_c(tmp_path):
    src = tmp_path / "styletts2_header.c"
    src.write_text('#include "fluidaudio_b200_styletts2.h"\n'
                   'int main(void) { int32_t b, r;\n'
                   '  (void)fa_styletts2_plan(10, &b, &r);\n'
                   '  return FA_STYLETTS2_STYLE_DIM + FA_STYLETTS2_REF_SPLIT + FA_STYLETTS2_NOISE_ROWS\n'
                   '    + FA_STYLETTS2_DEFAULT_TOKENS + FA_STYLETTS2_MAX_TOKENS + FA_STYLETTS2_TAIL_TRIM\n'
                   '    + FA_STYLETTS2_SAMPLE_RATE + FA_STYLETTS2_NONFINITE_DURATION; }\n')
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I",
                           os.path.join(ROOT, "include"), str(src)])


def test_the_documented_constants_are_the_kernels():
    text = open(HEADER).read()
    core = open(os.path.join(FAMILY, "styletts2_core.cuh")).read()
    for name, value in (("STYLE_DIM", 256), ("REF_SPLIT", 128), ("NOISE_ROWS", 5), ("DEFAULT_TOKENS", 57),
                        ("MAX_TOKENS", 256), ("TAIL_TRIM", 50), ("SAMPLE_RATE", 24000)):
        assert re.search(rf"#define FA_STYLETTS2_{name} {value}\b", text), name
    for decl in ("kStyleDim = 256;", "kRefSplit = 128;", "kNoiseRows = 5;", "kDefaultTokens = 57;",
                 "kMaxTokens = 256;", "kTailTrim = 50;"):
        assert decl in core, decl
    reasons = re.findall(r"FA_STYLETTS2_([A-Z_]+) = (\d+)", text)
    assert [int(v) for _, v in reasons] == list(range(4))
    assert re.findall(r"k(?:Ok|NoTokens|NoBucket|NonfiniteDuration) = (\d)", core) == ["0", "1", "2", "3"]
    # the noise is LuxTTS's one implementation, not a second SplitMix64
    assert "luxtts::gaussian_at" in core and "0x9E3779B97F4A7C15" not in core


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
        for m in re.finditer(r"\b(?:FA_API\s+fa_status|FA_STYLETTS2_API)\s+(\w+)\s*\(", code):
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
        exported |= set(re.findall(r"\bFA_(?:STYLETTS2_)?API\s+(?:\w+\s+)*?(fa_\w+)\s*\(", _code(os.path.join(FAMILY, name))))
    assert exported == set(REFUSED)


def test_every_launch_goes_through_the_counting_helpers():
    offenders = []
    for name in sorted(os.listdir(FAMILY)):
        code = re.sub(r"/\*.*?\*/|//[^\n]*", " ", open(os.path.join(FAMILY, name), encoding="utf-8").read(), flags=re.S)
        offenders += [f"{name}: {t}" for t in ("<<<", "cudaLaunchCooperativeKernel", "cudaLaunchKernel") if t in code]
        offenders += [f"{name}: {m}" for m in re.findall(r"\b(cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*)\s*\(", code)]
    assert not offenders
    assert "launch(" in open(os.path.join(FAMILY, "styletts2_kernels.cu")).read()


# ------------------------------------------------------------------------------------------------ refusals write nothing
def _sampler(L, sizes, bucket, seeds=None):
    n = len(sizes)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    ids = np.arange(max(int(off[-1]), 1), dtype=np.int32)
    sd = np.arange(n, dtype=np.uint64) if seeds is None else seeds
    tokens = np.full((n, max(bucket, 1)), 7, np.int32)
    mask, noise = tokens.copy(), np.full((n, 5, 256), 7, np.float32)
    reasons = np.full(n, -9, np.int32)
    st = L.fa_styletts2_sampler_inputs(i32(n), P(ids), P(off), P(sd), i32(bucket),
                                       P(tokens), P(mask), P(noise), P(reasons))
    untouched = (tokens == 7).all() and (mask == 7).all() and (noise == 7).all()
    return st, reasons, untouched


def test_sampler_refusals_set_reasons_and_write_nothing_else(lib):
    for sizes, bucket, want in (([5, 0, 3], 57, [0, 1, 0]), ([5, 257], 57, [0, 2]), ([300], 256, [2])):
        st, reasons, untouched = _sampler(lib, sizes, bucket)
        assert st == 1 and reasons.tolist() == want and untouched
        assert b"reason" in lib.fa_last_error()
    # a request of another bucket: reasons all 0, refused, nothing written
    for sizes, bucket in (([5, 58], 57), ([64, 65], 64), ([57], 64), ([200], 128)):
        st, reasons, untouched = _sampler(lib, sizes, bucket)
        assert st == 1 and reasons.tolist() == [0] * len(sizes) and untouched
        assert b"outside bucket" in lib.fa_last_error()
    for bucket in (0, 56, 100, 512):
        st, reasons, untouched = _sampler(lib, [3], bucket)
        assert st == 1 and (reasons == -9).all() and untouched and b"bucket" in lib.fa_last_error()
    off = np.array([3, 2], np.int64)
    r = np.full(1, -9, np.int32)
    assert lib.fa_styletts2_sampler_inputs(i32(1), N, P(off), P(off), i32(57), N, N, N,
                                           P(r)) == 1


def _align(L, counts, C_=4, lrow=None, lreq=None, dC=3, drow=None, dreq=None, tC=2, trow=None, treq=None, stride=64,
           device=False):
    counts = np.asarray(counts, np.int32)
    n, w = counts.size, int(counts.max())
    lrow, drow, trow = lrow or C_, drow or dC, trow or w
    lreq, dreq, treq = lreq or w * lrow, dreq or w * drow, treq or tC * trow
    logits = np.zeros(max(n * lreq, 1), np.float32)
    d, t = np.zeros(max(n * dreq, 1), np.float32), np.zeros(max(n * treq, 1), np.float32)
    en, asr = np.full(n * dC * stride, 7, np.float32), np.full(n * tC * stride, 7, np.float32)
    frames, durs, reasons = np.full(n, -9, np.int64), np.full(int(counts.sum()), -9, np.int32), np.full(n, -9, np.int32)
    fn = L.fa_styletts2_align_device if device else L.fa_styletts2_align
    st = fn(i32(n), P(counts), P(logits), i32(C_), i64(lrow), i64(lreq), P(d), i32(dC),
            i64(drow), i64(dreq), P(t), i32(tC), i64(trow), i64(treq), i64(stride), P(en),
            P(asr), P(frames), P(durs), P(reasons))
    untouched = (en == 7).all() and (asr == 7).all() and (frames == -9).all() and (durs == -9).all() and \
        (reasons == -9).all()
    return st, untouched


@pytest.mark.parametrize("device", [False, True])
def test_align_refusals_write_nothing(lib, device):
    cases = [dict(counts=[3, 0]), dict(counts=[257]), dict(counts=[3], C_=0), dict(counts=[3], dC=0),
             dict(counts=[3], tC=0), dict(counts=[3], stride=0), dict(counts=[3], stride=(1 << 22) + 1),
             dict(counts=[3], lrow=3), dict(counts=[3, 4], lreq=12), dict(counts=[3], drow=2),
             dict(counts=[3, 4], dreq=9), dict(counts=[3, 5], trow=4), dict(counts=[3], treq=5),
             dict(counts=[3], C_=(1 << 24) + 1), dict(counts=[3], dC=(1 << 20) + 1)]
    for kw in cases:
        st, untouched = _align(lib, device=device, **kw)
        assert st == 1 and untouched, kw
        assert lib.fa_last_error()
    assert lib.fa_styletts2_align(i32(-1), *ALIGN_NULLS) == 1 and b"count" in lib.fa_last_error()
    assert lib.fa_styletts2_align(i32(0), *ALIGN_NULLS) == 0   # nothing to do


def test_style_refusals(lib):
    one = np.zeros(256, np.float32)
    a = np.zeros(1, np.float32)
    out = np.full(128, 7, np.float32)
    for args in ((one, one, a, None, out, out), (one, None, a, a, out, out), (one, one, a, a, out, None)):
        ptrs = [None if x is None else P(x) for x in args]
        assert lib.fa_styletts2_style(i32(1), *ptrs) == 1 and (out == 7).all()
    assert lib.fa_styletts2_style(i32(0), N, N, N, N, N, N) == 0
    b, r = i32(-5), i32(-5)
    assert lib.fa_styletts2_plan(i32(-1), C.byref(b), C.byref(r)) == 1 and b.value == r.value == -5
