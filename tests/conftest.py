import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu on a machine that has one")


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure).  Builds liboracle.so on first use."""
    from oracle import oracle as O
    O.build()
    O.lib()
    return O


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def gpu_lib():
    """The CUDA library on a machine that has an H100; GPU tests fail (not skip) if it is unusable."""
    from fluidaudio_b200 import _lib
    L = _lib.load()
    assert _lib.device_count() >= 1, "no sm_90a device visible: GPU tests must run on a machine with an H100"
    return L
