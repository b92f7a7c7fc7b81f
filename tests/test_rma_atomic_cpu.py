"""The passive-target calls without a GPU: the numpy model (_rma_atomic_ref.py) pinned on hand-worked
cases (REPLACE and NO_OP, the f32 flush of a SUM whose fetch keeps the prior bits, the NaN rules of a
fetch, int64 wrap, compare-and-swap, serial fetches and lock-protected rounds), the facade's checks
(raised before the library is called), the answers before Init and in a control-plane-only world,
the ABI, and the C++ facade."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import _launch
import _rma_atomic_ref as A
import mpi_b200 as mpi
from _launch import assert_world_ok, run_world
from mpi_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "_rma_atomic_worker.py")
I64 = np.iinfo(np.int64)
TINY = np.float32(np.finfo(np.float32).tiny)


def bits(x):
    x = np.asarray(x)
    return x.view({4: np.uint32, 8: np.uint64}[x.dtype.itemsize]).tolist()


def test_replace_and_no_op():
    a = np.array([1.0, np.nan, -0.0], dtype=np.float64)
    b = np.array([np.nan, 2.0, 0.0], dtype=np.float64)
    old, new = A.fetch_op(a, b, A.REPLACE)
    assert bits(old) == bits(a) and bits(new) == bits(b)
    old, new = A.fetch_op(a, b, A.NO_OP)
    assert bits(old) == bits(a) and bits(new) == bits(a)
    old, new = A.fetch_op(a, None, A.NO_OP)                                   # NO_OP reads no origin
    assert bits(new) == bits(a)


def test_f32_sum_flushes_the_target_but_the_fetch_keeps_the_prior_bits():
    sub = np.float32(1e-39)
    a = np.array([sub, -sub, 1.5 * TINY, 1.0], dtype=np.float32)
    b = np.array([0.0, -0.0, -TINY, sub], dtype=np.float32)                 # -0 + -0 = -0; -0 + +0 would be +0
    old, new = A.fetch_op(a, b, A.SUM)
    assert bits(old) == bits(a)                                              # subnormals fetched as stored
    assert bits(new) == bits(np.array([0.0, -0.0, 0.0, 1.0], dtype=np.float32))


def test_nan_rules_of_a_fetch():
    payload = np.array([0x7FC01234], dtype=np.uint32).view(np.float32)[0]    # a NaN with a payload
    a = np.array([payload, 1.0, 5.0], dtype=np.float32)
    b = np.array([3.0, np.nan, 6.0], dtype=np.float32)
    for op in (A.MAX, A.MIN):
        old, new = A.fetch_op(a, b, op)
        assert bits(old) == bits(a)                                          # the NaN's own bits come back
        assert bits(new)[0] == 0x7FC01234 and new[1] == 1.0                  # a target NaN stays, an origin NaN is dropped
    assert A.fetch_op(a, b, A.MAX)[1][2] == 6.0 and A.fetch_op(a, b, A.MIN)[1][2] == 5.0
    old, new = A.fetch_op(a, b, A.SUM)
    assert bits(old) == bits(a) and np.isnan(new[0]) and np.isnan(new[1]) and new[2] == 11.0
    assert A.same_bits(new, np.array([np.nan, np.nan, 11.0], dtype=np.float32), nan_equal=True)
    assert not A.same_bits(new, np.array([np.nan, np.nan, 11.0], dtype=np.float32))


def test_int64_wrap_max_min_and_compare_and_swap():
    a = np.array([I64.max, I64.min, -1], dtype=np.int64)
    b = np.array([1, -1, I64.min], dtype=np.int64)
    assert A.fetch_op(a, b, A.SUM)[1].tolist() == [I64.min, I64.max, I64.max]
    assert A.fetch_op(a, b, A.MAX)[1].tolist() == [I64.max, -1, -1]
    assert A.fetch_op(a, b, A.MIN)[1].tolist() == [1, I64.min, I64.min]
    old, new = A.compare_and_swap([-1, 4, I64.min], 7, -1)
    assert old.tolist() == [-1, 4, I64.min] and new.tolist() == [7, 4, I64.min]


def test_serial_fetches_hand_out_every_ticket_once():
    fetched, final = A.serial(np.int64(0), [(A.SUM, 1)] * 5)
    assert [int(f) for f in fetched] == [0, 1, 2, 3, 4] and final == 5
    fetched, final = A.serial(np.float64(-1), [(A.REPLACE, 3.0), (A.REPLACE, 4.0), (A.NO_OP, 9.0)])
    assert fetched == [-1.0, 3.0, 4.0] and final == 4.0                      # a swap chain: fetched + final = all values


def test_locked_rounds():
    recs = A.locked_rounds(3, 2, 4, lambda k, r: [(k + r + j) % 3 for j in range(3)])
    assert [r.tolist() for r in recs] == [[6] * 4] * 3                       # n * R in every element
    recs = A.locked_rounds(2, 3, 2, lambda k, r: [0])
    assert recs[0].tolist() == [6, 6] and recs[1].tolist() == [0, 0]


class _Sized(mpi.Cuda):
    def Rank(self):
        return 1

    def Size(self):
        return 3


def test_facade_checks_before_the_library():
    w = mpi.Win(0)
    frozen = np.zeros(4)
    frozen.flags.writeable = False
    for call in (lambda: w.GetAccumulate(np.zeros(4), frozen, 0), lambda: w.GetAccumulate(np.zeros(3), b"abc", 0),
                 lambda: w.GetAccumulate(np.zeros(4), np.zeros(4, np.float32), 0),
                 lambda: w.GetAccumulate(np.zeros(4), mpi.DeviceSlice(4, np.float64, ptr=4096, owner=False), 0),
                 lambda: w.GetAccumulate(None, np.zeros(4), 0),                          # only NO_OP goes without an origin
                 lambda: w.GetAccumulate(np.zeros(2, mpi.LOC_F64), np.zeros(2, mpi.LOC_F64), 0),
                 lambda: w.FetchAndOp(True, 0), lambda: w.FetchAndOp(np.int32(1), 0), lambda: w.FetchAndOp("1", 0),
                 lambda: w.FetchAndOp(np.float16(1), 0), lambda: w.FetchAndOp(None, 0),
                 lambda: w.CompareAndSwap(1.0, 2, 0), lambda: w.CompareAndSwap(1, np.float64(2), 0),
                 lambda: w.CompareAndSwap(np.int32(1), 2, 0)):
        with pytest.raises(TypeError):
            call()
    for call in (lambda: w.GetAccumulate(np.zeros(4), np.zeros(3), 0), lambda: w.GetAccumulate(np.zeros(4), np.zeros(4), 0, -1),
                 lambda: w.FetchAndOp(1, 0, -1), lambda: w.CompareAndSwap(1, 2, 0, -3),
                 lambda: w.Lock(0, 0), lambda: w.Lock(0, 3), lambda: w.Lock(0, "exclusive")):
        with pytest.raises(ValueError):
            call()


def test_entries_before_init_report_not_initialised():
    lib = L.load()
    assert lib.b200mpi_size() == 0
    x = np.zeros(4, np.int64)
    p = x.ctypes.data
    for rc in (lib.b200mpi_win_lock(L.LOCK_EXCLUSIVE, 0, 0), lib.b200mpi_win_unlock(0, 0),
               lib.b200mpi_get_accumulate(p, p, 4, L.I64, L.SUM, 0, 0, 0, L.HOST), lib.b200mpi_fetch_and_op(p, p, L.I64, L.SUM, 0, 0, 0),
               lib.b200mpi_compare_and_swap(p, p, p, L.I64, 0, 0, 0), lib.b200mpi_compare_and_swap(p, p, p, L.F32, 0, 0, 0),
               lib.b200mpi_accumulate(p, 4, L.I64, L.REPLACE, 0, 0, 0, L.HOST)):
        assert rc == L.ERR_NOT_INIT
    w = mpi.Win(0)
    for call in (lambda: w.Lock(0), lambda: w.Lock(1, mpi.LOCK_SHARED), lambda: w.Unlock(0),
                 lambda: w.GetAccumulate(x, np.zeros(4, np.int64), 0), lambda: w.GetAccumulate(None, x, 0, op=mpi.NO_OP),
                 lambda: w.FetchAndOp(1, 0), lambda: w.FetchAndOp(1.5, 0, op=mpi.NO_OP), lambda: w.CompareAndSwap(1, 0, 0)):
        with pytest.raises(mpi.MpiError) as e:
            call()
        assert e.value.code == L.ERR_NOT_INIT


def test_header_binding_and_library_carry_the_entries():
    lib = ctypes.CDLL(mpi.LIB_PATH)
    with open(os.path.join(ROOT, "include", "b200mpi.h")) as f:
        header = f.read()
    for name, decl in (
            ("b200mpi_win_lock", "int b200mpi_win_lock(int lock_type, int target, int win);"),
            ("b200mpi_win_unlock", "int b200mpi_win_unlock(int target, int win);"),
            ("b200mpi_get_accumulate", "int b200mpi_get_accumulate(const void* origin, void* result, size_t count, int dtype, int op,\n"
                                       "                           int target, size_t target_disp, int win, int memkind);"),
            ("b200mpi_fetch_and_op", "int b200mpi_fetch_and_op(const void* origin, void* result, int dtype, int op,\n"
                                     "                         int target, size_t target_disp, int win);"),
            ("b200mpi_compare_and_swap", "int b200mpi_compare_and_swap(const void* origin, const void* compare, void* result, int dtype,\n"
                                         "                             int target, size_t target_disp, int win);")):
        assert name in L.SYMBOLS and hasattr(lib, name) and decl in header, name
    out = subprocess.run(["nm", "-D", "--defined-only", mpi.LIB_PATH], capture_output=True, text=True).stdout
    for name in ("b200mpi_win_lock", "b200mpi_win_unlock", "b200mpi_get_accumulate", "b200mpi_fetch_and_op", "b200mpi_compare_and_swap"):
        assert " T %s\n" % name in out, name
    for enum, value in (("B200MPI_REPLACE", 3), ("B200MPI_NO_OP", 4), ("B200MPI_LOCK_EXCLUSIVE", 1), ("B200MPI_LOCK_SHARED", 2)):
        assert "%s = %d" % (enum, value) in header, enum
    assert (L.REPLACE, L.NO_OP, L.LOCK_EXCLUSIVE, L.LOCK_SHARED) == (3, 4, 1, 2)
    assert (mpi.REPLACE, mpi.NO_OP, mpi.LOCK_EXCLUSIVE, mpi.LOCK_SHARED) == (3, 4, 1, 2)
    assert L.load().b200mpi_version() == 200


@pytest.mark.parametrize("n", [1, 2])
def test_control_plane_world_refuses_the_passive_target_calls(n, monkeypatch):
    monkeypatch.setattr(_launch, "WORKER", WORKER)
    assert_world_ok(run_world(n, "ra_control_only", args=["--control-only"], timeout=120))


def test_cpp_facade_rma_atomic():
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-rma-atomic-"), "rma_atomic_facade_test")
    lib = os.path.join(ROOT, "mpi_b200", "lib")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "rma_atomic_facade_test.cpp"),
                           "-L" + lib, "-lb200mpi", "-Wl,-rpath," + lib, "-pthread"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "rma atomic facade ok" in out.stdout, out.stdout + out.stderr
