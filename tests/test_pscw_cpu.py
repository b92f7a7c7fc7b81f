"""Generalized active target without a GPU: the header, binding and exported symbols of Post, Start,
Complete, Wait and Test; their answers before Init and in a control-plane-only world; the facade's
group checks (raised before the library is called); and the C++ facade."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import _launch
import mpi_b200 as mpi
from _launch import assert_world_ok, run_world
from mpi_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "_pscw_worker.py")
ENTRIES = ("b200mpi_win_post", "b200mpi_win_start", "b200mpi_win_complete", "b200mpi_win_wait", "b200mpi_win_test")


def test_header_binding_and_library_carry_the_entries():
    lib = ctypes.CDLL(mpi.LIB_PATH)
    with open(os.path.join(ROOT, "include", "b200mpi.h")) as f:
        header = f.read()
    for name, decl in (("b200mpi_win_post", "int b200mpi_win_post(const int* origins, int count, int win);"),
                       ("b200mpi_win_start", "int b200mpi_win_start(const int* targets, int count, int win);"),
                       ("b200mpi_win_complete", "int b200mpi_win_complete(int win);"),
                       ("b200mpi_win_wait", "int b200mpi_win_wait(int win);"),
                       ("b200mpi_win_test", "int b200mpi_win_test(int win, int* flag);")):
        assert name in L.SYMBOLS and hasattr(lib, name) and decl in header, name
    out = subprocess.run(["nm", "-D", "--defined-only", mpi.LIB_PATH], capture_output=True, text=True).stdout
    for name in ENTRIES:
        assert " T %s\n" % name in out, name
    version = header[header.index("#define B200MPI_VERSION"):header.index("#define B200MPI_MAX_RANKS")]
    for name in ("win_post", "win_start", "win_complete", "win_wait", "win_test"):
        assert name in version, name
    assert L.load().b200mpi_version() == 200


def test_entries_before_init_report_not_initialised():
    lib = L.load()
    assert lib.b200mpi_size() == 0
    grp = (ctypes.c_int * 2)(0, 1)
    flag = ctypes.c_int(9)
    for rc in (lib.b200mpi_win_post(grp, 2, 0), lib.b200mpi_win_start(grp, 2, 0), lib.b200mpi_win_post(None, 0, 0),
               lib.b200mpi_win_start(None, -1, 0), lib.b200mpi_win_complete(0), lib.b200mpi_win_wait(0),
               lib.b200mpi_win_test(0, ctypes.byref(flag)), lib.b200mpi_win_test(0, None)):
        assert rc == L.ERR_NOT_INIT
    assert flag.value == 9
    w = mpi.Win(0)
    for call in (lambda: w.Post([0]), lambda: w.Post([]), lambda: w.Start(np.array([0, 1])), lambda: w.Start(range(3)),
                 lambda: w.Post((np.int32(1), 2)), lambda: w.Complete(), lambda: w.Wait(), lambda: w.Test()):
        with pytest.raises(mpi.MpiError) as e:
            call()
        assert e.value.code == L.ERR_NOT_INIT


def test_facade_group_checks_before_the_library():
    w = mpi.Win(0)
    for bad in ([True], [0, False], [np.bool_(True)], [1.0], [np.float64(0)], ["0"], "01", [None], 3, None, [[0]],
                np.array([0.0, 1.0])):
        for call in (w.Post, w.Start):
            with pytest.raises(TypeError):
                call(bad)


@pytest.mark.parametrize("n", [1, 2])
def test_control_plane_world_refuses_pscw(n, monkeypatch):
    monkeypatch.setattr(_launch, "WORKER", WORKER)
    assert_world_ok(run_world(n, "pscw_control_only", args=["--control-only"], timeout=120))


def test_cpp_facade_pscw():
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-pscw-"), "pscw_facade_test")
    lib = os.path.join(ROOT, "mpi_b200", "lib")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "pscw_facade_test.cpp"),
                           "-L" + lib, "-lb200mpi", "-Wl,-rpath," + lib, "-pthread"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "pscw facade ok" in out.stdout, out.stdout + out.stderr
