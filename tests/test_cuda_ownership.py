"""Every CUDA buffer, stream and event of the library has an owner.

The owning types of ``fa_common.cuh`` (grow-only device / pinned buffers, stream and event owners and the descriptor
upload stage) are the only code under ``fluidaudio_b200/csrc/`` that allocates or frees device or pinned memory, or
creates or destroys a stream or an event, so a resource added anywhere else cannot be left without a release.  The
exception is the four C ABI entry points that hand memory to the caller and take it back.
"""
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from csrc_sources import CSRC, EXTENSIONS, path, sources  # noqa: E402

RESOURCE_CALL = re.compile(
    r"\b(cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|cudaStreamDestroy|cudaEventCreate\w*|cudaEventDestroy)\s*\(")
CALLER_MEMORY_ABI = ("fa_host_alloc", "fa_host_free", "fa_device_alloc", "fa_device_free")
SYNC_COPY = re.compile(r"\bcuda(Memcpy|Memset)(2D|3D|Peer|ToSymbol|FromSymbol|ToArray|FromArray)?\s*\(")
# the C ABI's caller-facing copies, synchronous by contract, and the copy-engine probe's scratch fill
SYNC_COPY_ALLOWED = ("fa_memcpy_h2d", "fa_memcpy_d2h", "fa_memcpy_probe")


def _code(path):
    """source text without comments"""
    with open(path, encoding="utf-8") as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    return re.sub(r"//[^\n]*", " ", text)


def _without_function(code, name):
    """`code` with the body of the function definition `name` removed (the function must be defined in it)"""
    m = re.search(r"\b" + name + r"\s*\([^;{]*\)\s*\{", code)
    assert m, f"{name} is not defined"
    depth, i = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(code[i], 0)
        i += 1
    return code[:m.end()] + code[i - 1:]


def test_the_scans_reach_every_family_directory():
    """every scan of csrc/ walks sources(), so none can silently drop a subdirectory again"""
    found = set(sources())
    families = sorted(d for d in os.listdir(CSRC) if os.path.isdir(os.path.join(CSRC, d)))
    assert {"ctc", "ctc_decode", "lseend", "online_diar", "vad"} <= set(families)
    for fam in families:
        for d, _, files in os.walk(os.path.join(CSRC, fam)):
            rel = os.path.relpath(d, CSRC).replace(os.sep, "/")
            want = {f"{rel}/{n}" for n in files if n.endswith(EXTENSIONS)}
            assert want <= found, (rel, want - found)


def test_cuda_resources_are_made_only_by_the_owning_types():
    offenders = []
    for name in sources():
        if name == "fa_common.cuh":
            continue
        code = _code(path(name))
        if name == "capi.cu":
            for fn in CALLER_MEMORY_ABI:
                code = _without_function(code, fn)
        offenders += [f"{name}: {m.group(1)}" for m in RESOURCE_CALL.finditer(code)]
    assert not offenders, f"CUDA resources made or released outside the owners of fa_common.cuh: {offenders}"


def test_no_synchronous_copy_or_fill():
    """A synchronous cudaMemcpy from pageable memory may return before the copy has landed, and it runs on the legacy
    stream, which the owners' non-blocking streams are not ordered after.  Uploads go on the stream of the kernels that
    read them (cudaMemcpyAsync, then that stream's synchronisation where the source does not outlive the call)."""
    offenders = []
    for name in sources():
        code = _code(path(name))
        if name == "capi.cu":
            for fn in SYNC_COPY_ALLOWED:
                code = _without_function(code, fn)
        code, owner = _scopes(code)
        offenders += [f"{name}: {owner[m.start()]}: {m.group(0)[:-1].strip()}" for m in SYNC_COPY.finditer(code)]
    assert not offenders, f"synchronous copies or fills: {offenders}"


OWNER_DECL = re.compile(r"\b(DeviceBuffer|PinnedBuffer|Stream)\b\s*(<[^;{}()]*?>)?\s*[A-Za-z_]\w*")
LOCAL_OWNERS_ALLOWED = {
    ("fa_common.cuh", "grow_slots"),
    ("capi.cu", "fa_memcpy_probe"),
    # grow_slots' twin for three per-slot arrays, one of them re-pitched to a new speaker capacity
    ("online_diar/online_diar_kernels.cu", "grow"),
}
THREAD_LOCALS_ALLOWED = {("capi.cu", "g_error"), ("capi.cu", "t_ev"), ("ahc_kernels.cu", "g_last_ms")}


def _scopes(code):
    """`code` without preprocessor lines and string / character literals, and for each of its characters the function
    whose body encloses it (None at namespace and class scope)"""
    code = re.sub(r"^[ \t]*#(?:[^\n]*\\\n)*[^\n]*", " ", code, flags=re.M)
    code = re.sub(r'"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', '""', code)
    owner, stack, start = [], [], 0   # stack: per open brace, the function whose body it opens or lies in
    for i, ch in enumerate(code):
        if ch == "{":
            head = code[start:i]
            if stack and stack[-1]:
                stack.append(stack[-1])
            elif re.search(r"\b(namespace|extern|struct|class|union|enum)\b", head):
                stack.append(None)
            else:
                m = re.search(r"(\w+)\s*\(", head)
                stack.append(m.group(1) if m else "?")
        elif ch == "}" and stack:
            stack.pop()
        if ch in "{};":
            start = i + 1
        owner.append(stack[-1] if stack else None)
    return code, owner


def test_handle_less_calls_own_no_stream_or_buffer_of_their_own():
    """A stream or buffer made inside a function body is made (and, for device memory, freed, which waits for the device)
    on every call; handle-less calls lease a pooled context (call_context.h) instead, and per-thread state would bypass
    that pool."""
    offenders = []
    for name in sources():
        code, owner = _scopes(_code(path(name)))
        for m in OWNER_DECL.finditer(code):
            fn = owner[m.start()]
            if fn and (name, fn) not in LOCAL_OWNERS_ALLOWED:
                offenders.append(f"{name}: {fn}: {' '.join(m.group(0).split())}")
        for m in re.finditer(r"\bthread_local\b([^;=\[{(]*)", code):
            var = re.findall(r"\w+", m.group(1))[-1]
            if (name, var) not in THREAD_LOCALS_ALLOWED:
                offenders.append(f"{name}: {owner[m.start()] or 'namespace scope'}: thread_local {var}")
    assert not offenders, f"streams or buffers inside function bodies, or thread_local state: {offenders}"


def test_the_owning_types_make_every_kind_of_resource():
    code = _code(path("fa_common.cuh"))
    for call in ("cudaMalloc", "cudaMallocHost", "cudaFree", "cudaFreeHost", "cudaStreamCreateWithFlags",
                 "cudaStreamDestroy", "cudaEventCreateWithFlags", "cudaEventDestroy"):
        assert re.search(r"\b" + call + r"\s*\(", code), call
