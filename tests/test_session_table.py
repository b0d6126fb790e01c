"""CPU tests of the session table the live log-mel streams and the Sortformer sessions keep their ids and host mirrors in
(``fluidaudio_b200/csrc/session_table.h``), compiled with g++ behind a small C shim (``tests/emul/session_table_shim.cpp``):

* open gives the lowest closed id, and a reopened id starts from a value-initialised session;
* a full table grows to the minimum slot count, then doubles, keeping every live session's mirror;
* a failed growth returns its status and leaves the slot count, the live flags and the mirrors as they were; a failed
  init leaves the id closed;
* check rejects negative, out-of-range, closed and repeated ids under the caller's error prefix;
* commit writes the listed sessions only.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "fluidaudio_b200", "csrc")
I32P = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
I64P = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
OK, INVALID, ALLOCATION_FAILURE, CUDA_ERROR = 0, 1, 4, 7   # FA_*


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("session_table") / "libsession_table.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-I", CSRC, "-o", out,
                           os.path.join(ROOT, "tests", "emul", "session_table_shim.cpp")])
    L = C.CDLL(out)
    vp, i32, pi32 = C.c_void_p, C.c_int32, C.POINTER(C.c_int32)
    L.st_create.restype = vp
    L.st_destroy.argtypes = [vp]
    L.st_last_error.restype = C.c_char_p
    L.st_slots.argtypes = [vp]
    L.st_valid.argtypes = [vp, i32]
    L.st_open.argtypes = [vp, i32, i32, i32, pi32, pi32, pi32]
    L.st_close.argtypes = [vp, i32, C.c_char_p]
    L.st_check.argtypes = [vp, i32, I32P, C.c_char_p]
    L.st_get.argtypes = [vp, i32, C.POINTER(C.c_longlong), pi32]
    L.st_set.argtypes = [vp, i32, C.c_longlong, i32]
    L.st_commit.argtypes = [vp, i32, I32P, I64P, I32P]
    return L


class Table:
    def __init__(self, L, min_slots):
        self.L, self.min_slots, self.t = L, min_slots, L.st_create()
        self.grows = []   # slot counts grow was called with

    def close_table(self):
        self.L.st_destroy(self.t)

    def open(self, grow_status=OK, init_status=OK):
        """(status, id, id init was called with)"""
        sid, grown, init = C.c_int32(-1), C.c_int32(), C.c_int32()
        st = self.L.st_open(self.t, self.min_slots, grow_status, init_status, C.byref(sid), C.byref(grown),
                            C.byref(init))
        if grown.value >= 0:
            self.grows.append(grown.value)
        return st, sid.value, init.value

    def close(self, sid, where=b"probe"):
        return self.L.st_close(self.t, sid, where)

    @property
    def slots(self):
        return self.L.st_slots(self.t)

    def live(self):
        return [s for s in range(self.slots) if self.L.st_valid(self.t, s)]

    def get(self, sid):
        v, tag = C.c_longlong(), C.c_int32()
        self.L.st_get(self.t, sid, C.byref(v), C.byref(tag))
        return v.value, tag.value

    def set(self, sid, value, tag):
        self.L.st_set(self.t, sid, value, tag)

    def mirrors(self):
        return [self.get(s) for s in range(self.slots)]

    def check(self, ids, where=b"probe push"):
        return self.L.st_check(self.t, len(ids), np.array(ids, np.int32), where)

    def commit(self, ids, values, tags):
        self.L.st_commit(self.t, len(ids), np.array(ids, np.int32), np.array(values, np.int64), np.array(tags, np.int32))


@pytest.fixture
def table(lib):
    t = Table(lib, 4)
    yield t
    t.close_table()


def test_lowest_closed_id_is_reused(table):
    assert [table.open()[1] for _ in range(6)] == list(range(6))
    for s in (4, 1, 2):
        table.set(s, 100 + s, s)
        assert table.close(s) == OK
    assert table.close(1) == INVALID                                   # closed twice
    assert table.open()[1:] == (1, 1)
    assert table.get(1) == (0, 0)                                      # value-initialised, whatever it held
    assert [table.open()[1] for _ in range(3)] == [2, 4, 6]
    assert table.live() == list(range(7))
    assert table.close(-1) == INVALID and table.close(table.slots) == INVALID


def test_growth_goes_min_then_doubling_and_keeps_the_live_sessions(table):
    for s in range(17):
        st, sid, init = table.open()
        assert (st, sid, init) == (OK, s, s)
        table.set(s, 1000 * s + 7, -s)
    assert table.grows == [4, 8, 16, 32]
    assert table.slots == 32
    assert table.mirrors()[:17] == [(1000 * s + 7, -s) for s in range(17)]
    assert table.live() == list(range(17))
    for s in range(17, 32):
        assert table.open()[1] == s
    assert table.grows == [4, 8, 16, 32]                               # no growth while a slot is free
    assert table.open()[1] == 32 and table.grows[-1] == 64
    # a larger minimum wins over doubling
    big = Table(table.L, 64)
    assert big.open()[1] == 0 and big.grows == [64]
    big.close_table()


@pytest.mark.parametrize("status", [ALLOCATION_FAILURE, CUDA_ERROR])
def test_failed_growth_leaves_the_table_as_it_was(table, status):
    for s in range(4):
        table.open()
        table.set(s, s * s + 1, 10 + s)
    table.close(2)
    assert table.open()[1] == 2                                        # a free slot: no growth, no failure
    before = (table.slots, table.live(), table.mirrors())
    st, sid, init = table.open(grow_status=status)
    assert (st, sid, init) == (status, -1, -1)
    assert table.grows[-1] == 8
    assert (table.slots, table.live(), table.mirrors()) == before
    assert table.open()[:2] == (OK, 4) and table.slots == 8            # the next growth succeeds where it left off


def test_failed_init_leaves_the_id_closed(table):
    assert [table.open()[1] for _ in range(3)] == [0, 1, 2]
    st, sid, init = table.open(init_status=CUDA_ERROR)
    assert (st, sid, init) == (CUDA_ERROR, -1, 3)
    assert table.live() == [0, 1, 2]
    assert table.open()[:2] == (OK, 3)


def test_check_rejects_bad_ids_under_the_callers_prefix(table, lib):
    for _ in range(5):
        table.open()
    table.close(3)
    assert table.check([]) == OK
    assert table.check([4, 0, 2, 1]) == OK
    cases = {
        (0, -1): "session -1 is not open",
        (0, 5): "session 5 is not open",                               # past the last live id
        (1, 8): "session 8 is not open",                               # past the slot count
        (2, 3): "session 3 is not open",                               # closed
        (0, 2, 0): "session 0 appears twice",
        (4, 1, 4): "session 4 appears twice",
    }
    for ids, text in cases.items():
        assert table.check(list(ids), b"mel stream push") == INVALID, ids
        assert lib.st_last_error().decode() == "mel stream push: " + text
    assert table.check([0, 3], b"sortformer update") == INVALID
    assert lib.st_last_error().decode() == "sortformer update: session 3 is not open"
    assert table.close(3, b"sortformer") == INVALID
    assert lib.st_last_error().decode() == "sortformer: session 3 is not open"


def test_commit_writes_only_the_listed_sessions(table):
    for s in range(6):
        table.open()
        table.set(s, s, s)
    table.commit([4, 1, 3], [40, 10, 30], [-4, -1, -3])
    assert table.mirrors()[:6] == [(0, 0), (10, -1), (2, 2), (30, -3), (40, -4), (5, 5)]
    table.commit([], [], [])
    assert table.mirrors()[:6] == [(0, 0), (10, -1), (2, 2), (30, -3), (40, -4), (5, 5)]
