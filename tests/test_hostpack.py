"""GPU-less checks of the host-side call helpers in okvis_b200/csrc/okb_hostpack.hpp: the buffer layout every
staging / scratch / arena buffer of the library uses (Carve), the runs of consecutive slots that commits and copies
are issued per (for_runs), and the host-thread spread of uploads, downloads and image packing (parallel_for)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def hp(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostpack") / "libhostpack_check.so")     # the source tree may be read-only
    subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-pthread", "-shared", "-o", so,
                           os.path.join(HERE, "hostcheck", "hostpack_check.cpp")])
    lib = C.CDLL(so)
    lib.hp_carve.restype = C.c_uint64
    lib.hp_parallel_for.restype = C.c_uint64
    return lib


def p(a):
    return C.c_void_p(a.ctypes.data)


def test_carve_layout(hp):
    """Each array starts where the previous one ended, rounded up to the alignment: the closed form of the window
    arena's layout (256 bytes) and of the marginalisation scratch and job payloads (16)."""
    rng = np.random.default_rng(6)
    for align in (16, 256):
        for n in (1, 2, 7, 40):
            sizes = rng.integers(0, 5000, n).astype(np.uint64)
            sizes[rng.random(n) < 0.2] = 0
            offs = np.zeros(n, np.uint64)
            total = hp.hp_carve(p(sizes), n, C.c_uint64(align), p(offs))
            o, want = 0, []
            for b in sizes.tolist():
                want.append(o)
                o = (o + b + align - 1) // align * align
            assert offs.tolist() == want and total == o


def test_for_runs(hp):
    """Runs of consecutive slots in list order, also for an unsorted list with gaps and repeats; the first failing
    callback ends the walk and its status is returned."""
    slots = np.array([3, 4, 5, 9, 1, 2, 2, 7, 8, 0], np.int32)
    runs = [(3, 3), (9, 1), (1, 2), (2, 1), (7, 2), (0, 1)]
    first, count, nr = np.zeros(10, np.int32), np.zeros(10, np.int32), C.c_int()
    for stop_at in (-1, 0, 2, 5):
        rc = hp.hp_for_runs(p(slots), len(slots), stop_at, p(first), p(count), C.byref(nr))
        want = runs if stop_at < 0 else runs[:stop_at + 1]
        assert rc == (0 if stop_at < 0 else 7)
        assert list(zip(first[:nr.value].tolist(), count[:nr.value].tolist())) == want
    assert hp.hp_for_runs(p(slots), 0, -1, p(first), p(count), C.byref(nr)) == 0 and nr.value == 0


@pytest.mark.parametrize("n,T", [(37, 1), (37, 37), (5, 8), (100, 8)])
def test_parallel_for(hp, n, T):
    """Every index exactly once; thread t of T runs the indices i = t mod T, so a caller may keep per-thread state at
    i % T (okb_window_upload_batch keeps each thread's first error there); T = 1 runs inline."""
    visits, owner = np.zeros(n, np.int32), np.zeros(n, np.uint64)
    caller = hp.hp_parallel_for(n, T, p(visits), p(owner))
    assert visits.tolist() == [1] * n
    if T == 1:
        assert set(owner.tolist()) == {caller}
    else:
        by_residue = [set(owner[r::T].tolist()) for r in range(min(n, T))]
        assert all(len(s) == 1 for s in by_residue)
        threads = set().union(*by_residue)
        assert len(threads) == min(n, T) and caller not in threads
