"""Gather, Scatter, Gatherv, Scatterv and Allgatherv without a GPU: the oracle against its numpy
twin, the facade's argument checks (raised before the library is called), the answers before Init
and in a control-plane-only world, and the C++ facade's resizing."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import _gather_oracle as G
import _launch
import mpi_b200 as mpi
from mpi_b200 import _lib as L
from oracle import oracle as O
from _launch import assert_world_ok, run_world

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GATHER_WORKER = os.path.join(ROOT, "tests", "_gather_worker.py")
NEW_ENTRIES = ("b200mpi_gather", "b200mpi_scatter", "b200mpi_gatherv", "b200mpi_scatterv", "b200mpi_allgatherv")


def _blocks(rng, dt, counts):
    if dt == np.uint8:
        return [rng.integers(0, 256, c, dtype=np.uint8) for c in counts]
    if dt == np.int64:
        return [rng.integers(-2**63, 2**63 - 1, c, dtype=np.int64) for c in counts]
    return [rng.standard_normal(c).astype(dt) for c in counts]


def _tables(rng, n):
    yield [0] * n
    yield [int(c) for c in rng.integers(0, 50, n)]
    single = [0] * n
    single[int(rng.integers(0, n))] = 37
    yield single
    yield [int(c) for c in rng.integers(0, 3, n)]  # mostly zeros and ones


@pytest.mark.parametrize("dt", [np.uint8, np.int64, np.float32, np.float64])
@pytest.mark.parametrize("n", range(1, 9))
def test_oracle_gatherv_scatterv_match_numpy_twin(n, dt):
    rng = np.random.default_rng(1000 * n + np.dtype(dt).itemsize)
    for counts in _tables(rng, n):
        ins = _blocks(rng, dt, counts)
        packed = G.gatherv(ins)
        assert packed.dtype == np.dtype(dt) and packed.size == sum(counts)
        assert np.array_equal(packed.view(np.uint8), G.gatherv_np(ins).view(np.uint8))
        for me in range(n):
            got = G.scatterv(packed, counts, me)
            assert np.array_equal(got.view(np.uint8), G.scatterv_np(packed, counts, me).view(np.uint8))
            assert np.array_equal(got.view(np.uint8), ins[me].view(np.uint8))  # Scatter(Gather(x)) == x


@pytest.mark.parametrize("n", range(1, 9))
def test_uniform_gather_is_allgather_on_root(n):
    rng = np.random.default_rng(n)
    ins = _blocks(rng, np.float64, [13] * n)
    assert np.array_equal(G.gatherv(ins), O.allgather(ins))


class _Sized(mpi.Cuda):
    """A world of 3 seen from rank 1, without a library: every check below must fire before a call."""

    def Rank(self):
        return 1

    def Size(self):
        return 3


def test_facade_checks_shapes_and_types_before_the_library():
    c = _Sized()
    a4, a12, a11 = np.zeros(4, np.float32), np.zeros(12, np.float32), np.zeros(11, np.float32)
    with pytest.raises(ValueError):
        c.Gather(a4, a11, 1)                               # root's recv must hold Size()*len(send)
    with pytest.raises(ValueError):
        c.Gather(a4, np.zeros(12, np.float64), 1)          # element types differ
    with pytest.raises(ValueError):
        c.Gather(a4, None, 1)                              # root needs a recv
    with pytest.raises(ValueError):
        c.Scatter(a11, a4, 1)                              # root's send must hold Size()*len(recv)
    with pytest.raises(ValueError):
        c.Scatter(np.zeros(12, np.int64), a4, 1)
    with pytest.raises(ValueError):
        c.Gatherv(a4, a12, 1, [4, 4])                      # counts of the wrong length
    with pytest.raises(ValueError):
        c.Gatherv(a4, a12, 1, [4, 5, 3])                   # counts[rank] != len(send)
    with pytest.raises(ValueError):
        c.Gatherv(a4, a12, 1, [4, 4, -1])
    with pytest.raises(ValueError):
        c.Gatherv(a4, np.zeros(12, np.int64), 1, [4, 4, 4])  # mixed dtype
    with pytest.raises(ValueError):
        c.Allgatherv(a4, np.zeros(12, np.float64), [4, 4, 4])
    with pytest.raises(ValueError):
        c.Allgatherv(a4, a12, [4, 4, 4, 4])
    with pytest.raises(ValueError):
        c.Allgatherv(a4, a12, [3, 3, 3])
    with pytest.raises(ValueError):
        c.Scatterv(a12, a4, [4, 4], 1)
    with pytest.raises(ValueError):
        c.Scatterv(a12, a4, [4, 4, 3], 1)                  # sum(counts) != len(send) on root
    with pytest.raises(ValueError):
        c.Scatterv(a12, np.zeros(4, np.float64), [4, 4, 4], 1)
    with pytest.raises(ValueError):
        c.Scatterv(a12, a4, None, 1)                       # root must pass counts
    with pytest.raises(ValueError):
        c.Scatterv(a12, None, [4, 4, 4], 1)
    dev = mpi.DeviceSlice(12, np.float32, ptr=4096, owner=False)
    with pytest.raises(ValueError):
        c.Gather(a4, dev, 1)                               # mixed memory kinds
    with pytest.raises(ValueError):
        c.Allgatherv(dev[0:4], a12, [4, 4, 4])
    with pytest.raises(ValueError):
        c.Allgatherv(dev[0:4], mpi.DeviceSlice(11, np.float32, ptr=4096, owner=False), [4, 4, 4])  # a device recv is never resized
    with pytest.raises(TypeError):
        c.Gather([1.0, 2.0], a12, 1)                       # not a typed buffer


def test_new_entries_before_init_report_not_initialised():
    lib = L.load()
    assert lib.b200mpi_size() == 0
    x = np.zeros(8, np.float32)
    tab = (ctypes.c_size_t * 2)(4, 4)
    rcs = [lib.b200mpi_gather(x.ctypes.data, x.ctypes.data, 4, L.F32, 0, L.HOST),
           lib.b200mpi_scatter(x.ctypes.data, x.ctypes.data, 4, L.F32, 0, L.HOST),
           lib.b200mpi_gatherv(x.ctypes.data, x.ctypes.data, tab, L.F32, 0, L.HOST),
           lib.b200mpi_scatterv(x.ctypes.data, x.ctypes.data, tab, L.F32, 0, L.HOST),
           lib.b200mpi_allgatherv(x.ctypes.data, x.ctypes.data, tab, L.F32, L.HOST)]
    assert rcs == [L.ERR_NOT_INIT] * 5
    for call in (lambda: mpi.Gather(x[:4], x, 0), lambda: mpi.Scatter(x, x[:4], 0), lambda: mpi.Gatherv(x[:4], x),
                 lambda: mpi.Scatterv(x, x[:4], [4, 4]), lambda: mpi.Allgatherv(x[:4])):
        with pytest.raises(mpi.MpiError) as e:
            call()
        assert e.value.code == L.ERR_NOT_INIT


def test_header_binding_and_library_carry_the_new_entries():
    lib = ctypes.CDLL(mpi.LIB_PATH)
    for name in NEW_ENTRIES:
        assert name in L.SYMBOLS and hasattr(lib, name)
    assert L.load().b200mpi_version() == 200


@pytest.mark.parametrize("n", [1, 2, 4])
def test_control_plane_world_refuses_the_new_entries(n, monkeypatch):
    monkeypatch.setattr(_launch, "WORKER", GATHER_WORKER)
    res = run_world(n, "gather_control_only", args=["--control-only"], timeout=120)
    assert_world_ok(res)


def test_cpp_facade_gather_resizing():
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-gather-"), "gather_facade_test")
    lib = os.path.join(ROOT, "mpi_b200", "lib")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "gather_facade_test.cpp"),
                           "-L" + lib, "-lb200mpi", "-Wl,-rpath," + lib, "-pthread"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "gather facade ok" in out.stdout, out.stdout + out.stderr
