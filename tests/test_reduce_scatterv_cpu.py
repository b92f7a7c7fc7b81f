"""ReduceScatterv without a GPU: the numpy restatement on hand-worked values and against the C oracle,
the host build of the kernel's (head, vectors, tail) split, the facade's argument checks (raised
before the library is called), the answers before Init and in a control-plane-only world, the ABI,
and the C++ facade."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import _launch
import _rsv_ref as V
import mpi_b200 as mpi
from _footprint_worker import gen_values
from _launch import assert_world_ok, run_world
from mpi_b200 import _lib as L
from oracle import oracle as O
from test_scan_cpu import same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RSV_WORKER = os.path.join(ROOT, "tests", "_rsv_worker.py")
nan, inf = np.nan, np.inf

# Three ranks, table [2, 0, 3]: rank 0 reduces elements 0-1, rank 1 nothing, rank 2 elements 2-4.
# Signed values, -0 meeting +0 in both orders, a NaN first and last in rank order, and +-Inf.
TABLE3 = [2, 0, 3]
X3 = [np.array([1.5, -0.0, 0.0, nan, inf]),
      np.array([-3.0, 0.0, -0.0, 1.0, -inf]),
      np.array([2.0, -1.0, nan, -1.0, 3.0])]
# worked by hand with b > a ? b : a, b < a ? b : a and a + b, left to right in rank order
HAND = {
    O.MAX: [[2.0, -0.0], [], [0.0, nan, inf]],
    O.MIN: [[-3.0, -1.0], [], [0.0, nan, -inf]],
    O.SUM: [[0.5, -1.0], [], [nan, nan, nan]],
}


@pytest.mark.parametrize("op", [O.SUM, O.MAX, O.MIN])
def test_restatement_matches_the_hand_worked_three_rank_table(op):
    got = V.rsv_np(X3, TABLE3, op)
    for j in range(3):
        assert same(got[j], np.array(HAND[op][j], dtype=np.float64)), (op, j, got[j])
        assert same(got[j], V.rsv_oracle(X3, TABLE3, op, j)), (op, j)


def test_restatement_wraps_i64_sums_like_go():
    big = np.iinfo(np.int64)
    xs = [np.array([big.max, big.min, -1]), np.array([1, -1, 7]), np.array([-5, big.max, big.min])]
    table = [1, 2, 0]
    got = V.rsv_np(xs, table, O.SUM)
    assert got[0].tolist() == [big.max - 4] and got[1].tolist() == [-2, big.min + 6] and got[2].size == 0
    assert V.rsv_np(xs, table, O.MAX)[1].tolist() == [big.max, 7]
    assert V.rsv_np(xs, table, O.MIN)[0].tolist() == [-5]
    for j in range(3):
        assert V.rsv_oracle(xs, table, O.SUM, j).tolist() == got[j].tolist()


def tables_for(n, rng):
    """Random, zero-entry (including a world whose every block is empty) and one-rank-heavy tables."""
    rand = [int(x) for x in rng.integers(0, 40, size=n)]
    zeros = [0 if r % 2 == 0 else int(x) for r, x in enumerate(rng.integers(1, 40, size=n))]
    return [rand, zeros, [0] * n, V.skewed(301, n), V.skewed(301, n, heavy=0), V.balanced(301, n)]


@pytest.mark.parametrize("dt", [np.float32, np.float64, np.int64])
@pytest.mark.parametrize("n", range(1, 9))
def test_restatement_matches_the_oracle(n, dt):
    rng = np.random.default_rng(7000 + n)
    for ti, table in enumerate(tables_for(n, rng)):
        xs = gen_values(dt, n, sum(table), 6000 + 10 * n + ti)
        for op in (O.SUM, O.MAX, O.MIN):
            got = V.rsv_np(xs, table, op)
            for j in range(n):
                assert got[j].size == table[j]
                assert same(got[j], V.rsv_oracle(xs, table, op, j)), (n, table, op, j)


@pytest.mark.parametrize("dt", [np.float32, np.float64, np.int64])
@pytest.mark.parametrize("n", range(1, 9))
def test_uniform_tables_match_oracle_reduce_scatter(n, dt):
    for c in (1, 5, 257):
        xs = gen_values(dt, n, n * c, 8000 + n * 7 + c)
        for op in (O.SUM, O.MAX, O.MIN):
            got = V.rsv_np(xs, [c] * n, op)
            for j in range(n):
                assert same(got[j], O.reduce_scatter(xs, j, op=op)), (n, c, op, j)


def test_block_split_covers_every_element_once():
    """split16 (kernels.cuh), compiled for the host: element sizes 1, 2, 4 and 8, every start residue,
    counts 0 ... 3 * EPV + 1 and a few large ones; vectors 16-byte aligned, each element covered once."""
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-split16-"), "split16_test")
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "split16_test.cu"), "-cudart", "static"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "split16 ok" in out.stdout, out.stdout + out.stderr


class _Sized(mpi.Cuda):
    """A world of 3 seen from rank 1, without a library: every check below must fire before a call."""

    def Rank(self):
        return 1

    def Size(self):
        return 3


def test_facade_checks_tables_and_buffers_before_the_library():
    c = _Sized()
    send = np.zeros(7, np.float32)
    recv = np.zeros(4, np.float32)
    dsend = mpi.DeviceSlice(7, np.float32, ptr=4096, owner=False)
    for counts in ([3, 4], [3, 4, 0, 0], [4, -1, 4]):              # table length, negative count
        with pytest.raises(ValueError):
            c.ReduceScatterv(send, recv, counts)
    with pytest.raises(ValueError):
        c.ReduceScatterv(send, recv, [2, 4, 2])                    # sum(counts) != len(send)
    with pytest.raises(ValueError):                                # counts[rank] != len(recv) (a device recv is not replaced)
        c.ReduceScatterv(dsend, mpi.DeviceSlice(3, np.float32, ptr=8192, owner=False), [2, 4, 1])
    with pytest.raises(ValueError):
        c.ReduceScatterv(send, np.zeros(4, np.float64), [2, 4, 1])  # element types differ
    with pytest.raises(ValueError):
        c.ReduceScatterv(send, mpi.DeviceSlice(4, np.float32, ptr=8192, owner=False), [2, 4, 1])  # memory kinds differ
    with pytest.raises(ValueError):
        c.ReduceScatterv(dsend, None, [2, 4, 1])                   # a device send needs a device recv
    with pytest.raises(ValueError):
        c.ReduceScatterv(send, None, None)                         # nothing to learn the table from
    with pytest.raises(TypeError):
        c.ReduceScatterv(np.zeros(7, np.int32), recv, [2, 4, 1])   # not a supported element type


def test_entries_before_init_report_not_initialised():
    lib = L.load()
    assert lib.b200mpi_size() == 0
    x = np.zeros(4, np.float32)
    table = (ctypes.c_size_t * 1)(4)
    assert lib.b200mpi_reduce_scatterv(x.ctypes.data, x.ctypes.data, table, L.F32, L.SUM, L.HOST) == L.ERR_NOT_INIT
    with pytest.raises(mpi.MpiError) as e:
        mpi.ReduceScatterv(x, x, [4])
    assert e.value.code == L.ERR_NOT_INIT


def test_header_binding_and_library_carry_the_entry():
    lib = ctypes.CDLL(mpi.LIB_PATH)
    assert "b200mpi_reduce_scatterv" in L.SYMBOLS and hasattr(lib, "b200mpi_reduce_scatterv")
    with open(os.path.join(ROOT, "include", "b200mpi.h")) as f:
        header = f.read()
    assert "int b200mpi_reduce_scatterv(const void* send, void* recv, const size_t* counts, int dtype, int op, int memkind);" in header
    assert L.load().b200mpi_version() == 200


@pytest.mark.parametrize("n", [1, 2])
def test_control_plane_world_refuses_reduce_scatterv(n, monkeypatch):
    monkeypatch.setattr(_launch, "WORKER", RSV_WORKER)
    assert_world_ok(run_world(n, "rsv_control_only", args=["--control-only"], timeout=120))


def test_cpp_facade_reduce_scatterv():
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-rsv-"), "reduce_scatterv_facade_test")
    lib = os.path.join(ROOT, "mpi_b200", "lib")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "reduce_scatterv_facade_test.cpp"),
                           "-L" + lib, "-lb200mpi", "-Wl,-rpath," + lib, "-pthread"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "reduce_scatterv facade ok" in out.stdout, out.stdout + out.stderr
