"""Alltoallv without a GPU: the table digest and displacements of kernels.cuh, the numpy
restatement on a hand-worked example, the facade's argument checks (raised before the library is
called), the answers before Init and in a control-plane-only world, and the C++ facade."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import _alltoallv_ref as A
import _launch
import mpi_b200 as mpi
from mpi_b200 import _lib as L
from oracle import oracle as O
from _launch import assert_world_ok, run_world

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALLTOALLV_WORKER = os.path.join(ROOT, "tests", "_alltoallv_worker.py")


def test_table_digest_and_displacements():
    """a2av_tables (kernels.cuh), compiled for the host: consistent matrices sum to 0, every single-entry
    change and every swap in one rank's row or column does not, displacements are prefix sums."""
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-a2av-"), "alltoallv_table_test")
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "alltoallv_table_test.cu"), "-cudart", "static"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "alltoallv table ok" in out.stdout, out.stdout + out.stderr


def test_restatement_hand_worked_3_ranks():
    m = [[1, 2, 0],
         [0, 1, 3],
         [2, 0, 1]]
    sends = [np.array([10, 11, 12], np.int64), np.array([20, 21, 22, 23], np.int64), np.array([30, 31, 32], np.int64)]
    assert A.alltoallv(sends, m, 0).tolist() == [10, 30, 31]
    assert A.alltoallv(sends, m, 1).tolist() == [11, 12, 20]
    assert A.alltoallv(sends, m, 2).tolist() == [21, 22, 23, 32]
    assert A.row(m, 1) == [0, 1, 3] and A.col(m, 1) == [2, 1, 0]


@pytest.mark.parametrize("n", range(1, 9))
def test_restatement_is_a_permutation_and_uniform_is_alltoall(n):
    for name, m in A.tables(n, 77 + n):
        sends = [np.arange(sum(m[i]), dtype=np.int64) + (i << 32) for i in range(n)]
        got = [A.alltoallv(sends, m, j) for j in range(n)]
        assert [g.size for g in got] == [sum(A.col(m, j)) for j in range(n)], name
        assert np.array_equal(np.sort(np.concatenate(got)), np.sort(np.concatenate(sends))), name
        if name == "uniform":
            for j in range(n):
                assert np.array_equal(got[j], O.alltoall(sends, j))
        if name == "quiet ranks":
            assert sum(m[0]) == 0 and got[n - 1].size == 0


class _Sized(mpi.Cuda):
    """A world of 3 seen from rank 1, without a library: every check below must fire before a call."""

    def Rank(self):
        return 1

    def Size(self):
        return 3


def test_facade_checks_shapes_and_types_before_the_library():
    c = _Sized()
    a6 = np.zeros(6, np.float32)
    with pytest.raises(ValueError):
        c.Alltoallv(a6, [3, 3], None, [1, 1, 1])                    # send table of the wrong length
    with pytest.raises(ValueError):
        c.Alltoallv(a6, [2, 2, 2], None, [1, 1])                    # recv table of the wrong length
    with pytest.raises(ValueError):
        c.Alltoallv(a6, [2, 5, -1], None, [1, 1, 1])                # negative count
    with pytest.raises(ValueError):
        c.Alltoallv(a6, [2, 2, 2], None, [1, -1, 1])
    with pytest.raises(ValueError):
        c.Alltoallv(a6, [2, 2, 1], None, [1, 1, 1])                 # sum(send_counts) != len(send)
    with pytest.raises(ValueError):
        c.Alltoallv(a6, [2, 2, 2], np.zeros(3, np.float64), [1, 1, 1])  # mixed dtype
    dev = mpi.DeviceSlice(6, np.float32, ptr=4096, owner=False)
    with pytest.raises(ValueError):
        c.Alltoallv(a6, [2, 2, 2], dev[0:3], [1, 1, 1])             # mixed memory kinds
    with pytest.raises(ValueError):
        c.Alltoallv(dev, [2, 2, 2], a6[:3], [1, 1, 1])
    with pytest.raises(ValueError):
        c.Alltoallv(dev, [2, 2, 2], mpi.DeviceSlice(4, np.float32, ptr=8192, owner=False), [1, 1, 1])  # a device recv is never resized
    with pytest.raises(ValueError):
        c.Alltoallv(dev, [2, 2, 2], None, [1, 1, 1])                # a device send needs a device recv
    with pytest.raises(TypeError):
        c.Alltoallv([1.0, 2.0], [1, 1, 0], None, [1, 1, 1])          # not a typed buffer


def test_alltoallv_before_init_reports_not_initialised():
    lib = L.load()
    assert lib.b200mpi_size() == 0
    x = np.zeros(8, np.float32)
    tab = (ctypes.c_size_t * 2)(4, 4)
    assert lib.b200mpi_alltoallv(x.ctypes.data, tab, x.ctypes.data, tab, L.F32, L.HOST) == L.ERR_NOT_INIT
    for call in (lambda: mpi.Alltoallv(x, [4, 4], np.zeros(8, np.float32), [4, 4]), lambda: mpi.Alltoallv(x, [4, 4])):
        with pytest.raises(mpi.MpiError) as e:
            call()
        assert e.value.code == L.ERR_NOT_INIT


def test_header_binding_and_library_carry_alltoallv():
    lib = ctypes.CDLL(mpi.LIB_PATH)
    assert "b200mpi_alltoallv" in L.SYMBOLS and hasattr(lib, "b200mpi_alltoallv")
    with open(os.path.join(ROOT, "include", "b200mpi.h")) as f:
        assert "int b200mpi_alltoallv(" in f.read()
    assert L.load().b200mpi_version() == 200


@pytest.mark.parametrize("n", [1, 2, 4])
def test_control_plane_world_refuses_alltoallv(n, monkeypatch):
    monkeypatch.setattr(_launch, "WORKER", ALLTOALLV_WORKER)
    res = run_world(n, "alltoallv_control_only", args=["--control-only"], timeout=120)
    assert_world_ok(res)


def test_cpp_facade_alltoallv_resizing_and_learning():
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-a2av-"), "alltoallv_facade_test")
    lib = os.path.join(ROOT, "mpi_b200", "lib")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "alltoallv_facade_test.cpp"),
                           "-L" + lib, "-lb200mpi", "-Wl,-rpath," + lib, "-pthread"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "alltoallv facade ok" in out.stdout, out.stdout + out.stderr
