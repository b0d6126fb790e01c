"""Every CUDA buffer, stream and event of the library has an owner.

The owning types of ``fa_common.cuh`` (grow-only device / pinned buffers, stream and event owners and the descriptor
upload stage) are the only code under ``fluidaudio_b200/csrc/`` that allocates or frees device or pinned memory, or
creates or destroys a stream or an event, so a resource added anywhere else cannot be left without a release.  The
exception is the four C ABI entry points that hand memory to the caller and take it back.
"""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "fluidaudio_b200", "csrc")

RESOURCE_CALL = re.compile(
    r"\b(cudaMalloc\w*|cudaFree\w*|cudaStreamCreate\w*|cudaStreamDestroy|cudaEventCreate\w*|cudaEventDestroy)\s*\(")
CALLER_MEMORY_ABI = ("fa_host_alloc", "fa_host_free", "fa_device_alloc", "fa_device_free")


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


def test_cuda_resources_are_made_only_by_the_owning_types():
    offenders = []
    for name in sorted(os.listdir(CSRC)):
        if not name.endswith((".cu", ".cuh", ".h", ".cpp")) or name == "fa_common.cuh":
            continue
        code = _code(os.path.join(CSRC, name))
        if name == "capi.cu":
            for fn in CALLER_MEMORY_ABI:
                code = _without_function(code, fn)
        offenders += [f"{name}: {m.group(1)}" for m in RESOURCE_CALL.finditer(code)]
    assert not offenders, f"CUDA resources made or released outside the owners of fa_common.cuh: {offenders}"


def test_the_owning_types_make_every_kind_of_resource():
    code = _code(os.path.join(CSRC, "fa_common.cuh"))
    for call in ("cudaMalloc", "cudaMallocHost", "cudaFree", "cudaFreeHost", "cudaStreamCreateWithFlags",
                 "cudaStreamDestroy", "cudaEventCreateWithFlags", "cudaEventDestroy"):
        assert re.search(r"\b" + call + r"\s*\(", code), call
