"""One-sided communication without a GPU: the numpy model of a fence epoch on a hand-worked 3-rank
case and on the element rules (i64 wrap and exact MAX / MIN, f32 flush, float MAX / MIN and NaN), the facade's checks
(raised before the library is called), the answers before Init and in a control-plane-only world,
the ABI, and the C++ facade."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import _launch
import _rma_ref as R
import mpi_b200 as mpi
from _launch import assert_world_ok, run_world
from mpi_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RMA_WORKER = os.path.join(ROOT, "tests", "_rma_worker.py")
I64 = np.iinfo(np.int64)
TINY = np.float32(np.finfo(np.float32).tiny)


def f64_window(vals):
    return np.array(vals, dtype=np.float64).view(np.uint8)


def test_model_on_a_hand_worked_three_rank_epoch():
    # windows: rank 0 five f64, rank 1 two, rank 2 none
    E = R.Epoch([f64_window([1, 1, 1, 1, 7]), f64_window([0, 0]), np.empty(0, np.uint8)])
    E.put(np.array([10.0, 20.0]), 1, 0)                                    # rank 0 -> rank 1
    E.accumulate(np.array([1.0, 2.0]), 0, 1, R.SUM)                        # rank 1 -> rank 0 [1, 2]
    E.accumulate(np.array([3.0, 4.0]), 0, 2, R.SUM)                        # rank 2 -> rank 0 [2, 3]: overlaps at 2
    got = E.get(np.float64, 1, 0, 4)                                       # rank 2 reads rank 0's untouched element
    E.accumulate(np.array([5.0]), 0, 2, R.MAX)                             # then MAX over the sums already applied
    w = E.fence()
    assert got.tolist() == [7.0]
    assert w[0].view(np.float64).tolist() == [1.0, 2.0, 6.0, 5.0, 7.0]
    assert w[1].view(np.float64).tolist() == [10.0, 20.0]
    assert w[2].size == 0


def test_get_reads_the_window_at_the_opening_fence():
    E = R.Epoch([f64_window([1, 2, 3])])
    E.put(np.array([9.0]), 0, 1)
    assert E.get(np.float64, 3, 0, 0).tolist() == [1.0, 2.0, 3.0]
    assert E.fence()[0].view(np.float64).tolist() == [1.0, 9.0, 3.0]
    with pytest.raises(AssertionError):
        E.put(np.array([1.0, 2.0]), 0, 2)                                  # past the window


def test_i64_sum_wraps_and_max_min_are_exact():
    a = np.array([I64.max, I64.min, -1, 5], dtype=np.int64)
    b = np.array([1, -1, I64.min, I64.max], dtype=np.int64)
    assert R.combine(a, b, R.SUM).tolist() == [I64.min, I64.max, I64.max, I64.min + 4]
    assert R.combine(a, b, R.MAX).tolist() == [I64.max, -1, -1, I64.max]
    assert R.combine(a, b, R.MIN).tolist() == [1, I64.min, I64.min, 5]


def test_f32_sum_flushes_subnormal_inputs_and_results():
    sub = np.float32(1e-39)
    a = np.array([0.0, sub, 1.5 * TINY, -sub, -1.5 * TINY, 1.0, 2.0, -2.0], dtype=np.float32)
    b = np.array([2.0 ** -140, 0.0, -TINY, 0.0, TINY, 2.0 ** -140, -sub, 3.0], dtype=np.float32)
    want = np.array([0.0, 0.0, 0.0, 0.0, -0.0, 1.0, 2.0, 1.0], dtype=np.float32)
    assert np.array_equal(R.combine(a, b, R.SUM).view(np.uint32), want.view(np.uint32))
    # f64 keeps subnormals
    d = np.array([5e-324, 0.0])
    assert np.array_equal(R.combine(d, np.array([0.0, 5e-324]), R.SUM), [5e-324, 5e-324])


def test_float_max_min_keep_a_target_nan_and_drop_a_contribution_nan():
    for dt in (np.float32, np.float64):
        a = np.array([np.nan, 1.0, -5.0, 0.0], dtype=dt)
        b = np.array([3.0, np.nan, -6.0, -0.0], dtype=dt)
        mx, mn = R.combine(a, b, R.MAX), R.combine(a, b, R.MIN)
        assert np.isnan(mx[0]) and mx[1] == 1.0 and mx[2] == -5.0 and not np.signbit(mx[3])
        assert np.isnan(mn[0]) and mn[1] == 1.0 and mn[2] == -6.0 and not np.signbit(mn[3])  # -0 < +0 is false


class _Sized(mpi.Cuda):
    """A world of 3 seen from rank 1, without a library: every check below must fire before a call."""

    def Rank(self):
        return 1

    def Size(self):
        return 3


def test_facade_checks_before_the_library():
    c = _Sized()
    with pytest.raises(TypeError):
        c.WinCreate(np.zeros(4))                                           # a window is heap memory
    with pytest.raises(TypeError):
        c.WinCreate([1.0])
    w = mpi.Win(0)
    pairs = np.zeros(2, mpi.LOC_F64)
    dev_pairs = mpi.DeviceSlice(2, mpi.LOC_F32, ptr=4096, owner=False)
    frozen = np.zeros(4)
    frozen.flags.writeable = False                                         # Get must not write read-only memory
    for call in (lambda: w.Put(pairs, 0), lambda: w.Get(pairs, 0), lambda: w.Accumulate(dev_pairs, 0),
                 lambda: w.Put([1.0], 0), lambda: w.Get("abc", 0), lambda: w.Get(b"abc", 0),
                 lambda: w.Put(np.zeros(3, np.int32), 0), lambda: w.Get(memoryview(b"abcdefgh"), 0),
                 lambda: w.Get(frozen, 0)):
        with pytest.raises(TypeError):
            call()
    for call in (lambda: w.Put(np.zeros(3), 0, -1), lambda: w.Get(np.zeros(3), 2, -5), lambda: w.Accumulate(np.zeros(3), 1, -1),
                 lambda: w.Put(np.zeros(8)[::2], 0)):
        with pytest.raises(ValueError):
            call()


def test_entries_before_init_report_not_initialised():
    lib = L.load()
    assert lib.b200mpi_size() == 0
    x = np.zeros(4)
    wc = ctypes.c_int(-1)
    for rc in (lib.b200mpi_win_create(None, 0, ctypes.byref(wc)), lib.b200mpi_win_free(0), lib.b200mpi_win_fence(0),
               lib.b200mpi_put(x.ctypes.data, 4, L.F64, 0, 0, 0, L.HOST), lib.b200mpi_get(x.ctypes.data, 4, L.F64, 0, 0, 0, L.HOST),
               lib.b200mpi_accumulate(x.ctypes.data, 4, L.F64, L.SUM, 0, 0, 0, L.HOST)):
        assert rc == L.ERR_NOT_INIT
    w = mpi.Win(0)
    for call in (lambda: mpi.WinCreate(None), lambda: w.Put(x, 0), lambda: w.Get(x, 0), lambda: w.Accumulate(x, 0), w.Fence, w.Free):
        with pytest.raises(mpi.MpiError) as e:
            call()
        assert e.value.code == L.ERR_NOT_INIT


def test_header_binding_and_library_carry_the_entries():
    lib = ctypes.CDLL(mpi.LIB_PATH)
    with open(os.path.join(ROOT, "include", "b200mpi.h")) as f:
        header = f.read()
    for name, decl in (
            ("b200mpi_win_create", "int b200mpi_win_create(void* base, size_t bytes, int* win);"),
            ("b200mpi_win_free", "int b200mpi_win_free(int win);"),
            ("b200mpi_win_fence", "int b200mpi_win_fence(int win);"),
            ("b200mpi_put", "int b200mpi_put(const void* origin, size_t count, int dtype, int target, size_t target_disp, int win, int memkind);"),
            ("b200mpi_get", "int b200mpi_get(void* origin, size_t count, int dtype, int target, size_t target_disp, int win, int memkind);"),
            ("b200mpi_accumulate",
             "int b200mpi_accumulate(const void* origin, size_t count, int dtype, int op, int target, size_t target_disp, int win, int memkind);")):
        assert name in L.SYMBOLS and hasattr(lib, name) and decl in header, name
    assert L.load().b200mpi_version() == 200


@pytest.mark.parametrize("n", [1, 2])
def test_control_plane_world_refuses_the_rma_calls(n, monkeypatch):
    monkeypatch.setattr(_launch, "WORKER", RMA_WORKER)
    assert_world_ok(run_world(n, "rma_control_only", args=["--control-only"], timeout=120))


def test_cpp_facade_rma():
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-rma-"), "rma_facade_test")
    lib = os.path.join(ROOT, "mpi_b200", "lib")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "rma_facade_test.cpp"),
                           "-L" + lib, "-lb200mpi", "-Wl,-rpath," + lib, "-pthread"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "rma facade ok" in out.stdout, out.stdout + out.stderr
