"""The C++ / CUDA sources under ``fluidaudio_b200/csrc/``, its family subdirectories included, for the static checks
(test infrastructure).  Paths are relative to ``csrc/`` with ``/`` separators, so an allow-list names a file as
``online_diar/online_diar_kernels.cu``."""
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "fluidaudio_b200", "csrc")
EXTENSIONS = (".cu", ".cuh", ".h", ".cpp")


def sources():
    """every source under csrc/, recursively, sorted"""
    out = []
    for d, dirs, files in os.walk(CSRC):
        dirs.sort()
        rel = os.path.relpath(d, CSRC)
        out += [n if rel == "." else f"{rel}/{n}".replace(os.sep, "/") for n in files if n.endswith(EXTENSIONS)]
    return sorted(out)


def path(rel):
    return os.path.join(CSRC, *rel.split("/"))

