"""Scan and Exscan without a GPU: the numpy restatement of the rank-order prefix on hand-worked values
and against the C oracle, the facade's argument checks (raised before the library is called), the
answers before Init and in a control-plane-only world, and the C++ facade."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import _launch
import _scan_ref as S
import mpi_b200 as mpi
from _footprint_worker import gen_values
from _launch import assert_world_ok, run_world
from mpi_b200 import _lib as L
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCAN_WORKER = os.path.join(ROOT, "tests", "_scan_worker.py")
nan, inf = np.nan, np.inf

# Three ranks, one column per case: signed values, -0 meeting +0 in both orders, a NaN first and
# later in rank order, and +-Inf.
X3 = [np.array([1.5, -0.0, 0.0, nan, 1.0, inf]),
      np.array([-3.0, 0.0, -0.0, 1.0, nan, -inf]),
      np.array([2.0, -1.0, -0.0, -1.0, 2.0, 3.0])]
# prefix r on rank r, worked by hand with b > a ? b : a, b < a ? b : a and a + b, left to right
HAND = {
    O.MAX: [[1.5, -0.0, 0.0, nan, 1.0, inf], [1.5, -0.0, 0.0, nan, 1.0, inf], [2.0, -0.0, 0.0, nan, 2.0, inf]],
    O.MIN: [[1.5, -0.0, 0.0, nan, 1.0, inf], [-3.0, -0.0, 0.0, nan, 1.0, -inf], [-3.0, -1.0, 0.0, nan, 1.0, -inf]],
    O.SUM: [[1.5, -0.0, 0.0, nan, 1.0, inf], [-1.5, 0.0, 0.0, nan, nan, nan], [0.5, -1.0, 0.0, nan, nan, nan]],
}


def same(got, want):
    """Bit for bit, except that any NaN matches any NaN (sums make new NaNs)."""
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype.kind != "f":
        return np.array_equal(got.view(np.uint8), want.view(np.uint8))
    nan_g, nan_w = np.isnan(got), np.isnan(want)
    return np.array_equal(nan_g, nan_w) and np.array_equal(got[~nan_g].view(np.uint8), want[~nan_w].view(np.uint8))


@pytest.mark.parametrize("op", [O.SUM, O.MAX, O.MIN])
def test_restatement_matches_the_hand_worked_three_rank_prefixes(op):
    scan, ex = S.scan_np(X3, op), S.scan_np(X3, op, exclusive=True)
    for r in range(3):
        assert same(scan[r], np.array(HAND[op][r])), (op, r, scan[r])
    assert ex[0] is None
    for r in (1, 2):
        assert same(ex[r], np.array(HAND[op][r - 1])), (op, r, ex[r])


def test_restatement_wraps_i64_sums_like_go():
    big = np.iinfo(np.int64)
    xs = [np.array([big.max, big.min, -1]), np.array([1, -1, 7]), np.array([-5, big.max, big.min])]
    scan = S.scan_np(xs, O.SUM)
    assert scan[1].tolist() == [big.min, big.max, 6]
    assert scan[2].tolist() == [big.max - 4, -2, big.min + 6]
    assert S.scan_np(xs, O.MAX)[2].tolist() == [big.max, big.max, 7]
    assert S.scan_np(xs, O.MIN, exclusive=True)[2].tolist() == [1, big.min, -1]


@pytest.mark.parametrize("dt", [np.float32, np.float64, np.int64])
@pytest.mark.parametrize("n", range(1, 9))
def test_restatement_matches_oracle_prefixes(n, dt):
    xs = gen_values(dt, n, 301, 5000 + n)
    for op in (O.SUM, O.MAX, O.MIN):
        scan, ex = S.scan_np(xs, op), S.scan_np(xs, op, exclusive=True)
        for r in range(n):
            assert same(scan[r], S.scan_oracle(xs, op, r)), (n, op, r)
            want = S.scan_oracle(xs, op, r, exclusive=True)
            assert (ex[r] is None) == (want is None) and (want is None or same(ex[r], want)), (n, op, r)
            if r >= 1:  # Scan = combine(Exscan, x_r)
                assert same(scan[r], S.apply(op, ex[r], xs[r]))
        assert same(scan[n - 1], O.allreduce(xs, op, O.ORDER_RANK))


class _Sized(mpi.Cuda):
    """A world of 3 seen from rank 1, without a library: every check below must fire before a call."""

    def Rank(self):
        return 1

    def Size(self):
        return 3


def test_facade_checks_shapes_and_types_before_the_library():
    c = _Sized()
    a4 = np.zeros(4, np.float32)
    dev = mpi.DeviceSlice(4, np.float32, ptr=4096, owner=False)
    for fn in (c.Scan, c.Exscan):
        with pytest.raises(ValueError):
            fn(a4, np.zeros(5, np.float32))                # lengths differ
        with pytest.raises(ValueError):
            fn(a4, np.zeros(4, np.float64))                # element types differ
        with pytest.raises(ValueError):
            fn(a4, dev)                                    # memory kinds differ
        with pytest.raises(TypeError):
            fn([1.0, 2.0], a4)                             # not a typed buffer
        with pytest.raises(TypeError):
            fn(np.zeros(4, np.int32), np.zeros(4, np.int32))
    with pytest.raises(TypeError):
        c.Scan(a4, None)                                   # only Exscan takes a missing recv


def test_entries_before_init_report_not_initialised():
    lib = L.load()
    assert lib.b200mpi_size() == 0
    x = np.zeros(4, np.float32)
    assert lib.b200mpi_scan(x.ctypes.data, x.ctypes.data, 4, L.F32, L.SUM, L.HOST) == L.ERR_NOT_INIT
    assert lib.b200mpi_exscan(x.ctypes.data, None, 4, L.F32, L.SUM, L.HOST) == L.ERR_NOT_INIT
    for call in (lambda: mpi.Scan(x, x), lambda: mpi.Exscan(x, None, mpi.MAX)):
        with pytest.raises(mpi.MpiError) as e:
            call()
        assert e.value.code == L.ERR_NOT_INIT


def test_header_binding_and_library_carry_the_entries():
    lib = ctypes.CDLL(mpi.LIB_PATH)
    for name in ("b200mpi_scan", "b200mpi_exscan"):
        assert name in L.SYMBOLS and hasattr(lib, name)
    with open(os.path.join(ROOT, "include", "b200mpi.h")) as f:
        header = f.read()
    assert "int b200mpi_scan(const void* send, void* recv, size_t count, int dtype, int op, int memkind);" in header
    assert "int b200mpi_exscan(const void* send, void* recv, size_t count, int dtype, int op, int memkind);" in header
    assert L.load().b200mpi_version() == 200


@pytest.mark.parametrize("n", [1, 2])
def test_control_plane_world_refuses_scan(n, monkeypatch):
    monkeypatch.setattr(_launch, "WORKER", SCAN_WORKER)
    assert_world_ok(run_world(n, "scan_control_only", args=["--control-only"], timeout=120))


def test_cpp_facade_scan():
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-scan-"), "scan_facade_test")
    lib = os.path.join(ROOT, "mpi_b200", "lib")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "scan_facade_test.cpp"),
                           "-L" + lib, "-lb200mpi", "-Wl,-rpath," + lib, "-pthread"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "scan facade ok" in out.stdout, out.stdout + out.stderr
