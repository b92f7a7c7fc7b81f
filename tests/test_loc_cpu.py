"""AllreduceLoc and ReduceLoc (MAXLOC / MINLOC) without a GPU: the numpy restatement on hand-worked
3-rank cases and against the C oracle, the independence of the result from the bracketing, a host
build of the kernel's own ops, the facade's argument checks (raised before the library is called),
the answers before Init and in a control-plane-only world, the ABI, and the C++ facade."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import _launch
import _loc_oracle as LO
import _loc_ref as R
import mpi_b200 as mpi
from _launch import assert_world_ok, run_world
from mpi_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOC_WORKER = os.path.join(ROOT, "tests", "_loc_worker.py")
MAX, MIN = mpi.MAX, mpi.MIN
nan, inf = np.nan, np.inf
I64 = np.iinfo(np.int64)


def qnan(dn, payload):
    if dn == "f32":
        return np.array([0x7FC00000 | payload], dtype=np.uint32).view(np.float32)[0]
    return np.array([0x7FF8000000000000 | payload], dtype=np.uint64).view(np.float64)[0]


# Hand-worked cases over three ranks: (values per rank, locs per rank, f32 padding per rank or None,
# the rank whose pair wins).  Each case is one element; a dtype's cases run as one call.
HAND = {
    ("f64", MAX): [
        ([5.0, 5.0, 3.0], [4, 2, 9], None, 1),               # equal values: the smaller loc
        ([5.0, 5.0, 5.0], [2, 2, 1], None, 2),               # ... from any rank
        ([-0.0, 0.0, -0.0], [5, 5, 1], None, 2),             # -0 == +0: loc decides, rank 2's -0 is kept
        ([0.0, -0.0, 0.0], [3, 3, 3], None, 0),              # all equal: rank 0's +0
        ([1.0, inf, -inf], [0, 1, 2], None, 1),
        ([1.0, qnan("f64", 1), inf], [0, 5, 1], None, 1),    # NaN beats +Inf under MAX
        ([qnan("f64", 1), 1.0, qnan("f64", 3)], [4, 0, 2], None, 2),  # NaNs are equal: the smaller loc
        ([qnan("f64", 1), qnan("f64", 2), 7.0], [2, 2, 2], None, 0),  # ... and on a loc tie the lower rank
    ],
    ("f64", MIN): [
        ([1.0, 1.0, 1.0], [3, -1, -1], None, 1),
        ([-0.0, 0.0, 2.0], [4, 4, -7], None, 0),
        ([0.0, -0.0, 2.0], [4, 3, -7], None, 1),
        ([1.0, inf, -inf], [0, 1, 2], None, 2),
        ([-inf, qnan("f64", 9), 0.0], [0, 1, 2], None, 1),   # NaN beats -Inf under MIN too
        ([-inf, -inf, qnan("f64", 9)], [0, -4, 8], None, 2),
    ],
    ("f32", MAX): [
        ([2.0, 2.0, 2.0], [7, 7, 7], [0xAAAAAAAA, 0xBBBBBBBB, 0xCCCCCCCC], 0),  # full tie: rank 0's padding
        ([1.0, 2.0, 2.0], [0, 3, 3], [0x11111111, 0x22222222, 0x33333333], 1),
        ([1.0, 2.0, 2.0], [0, 3, -3], [0x11111111, 0x22222222, 0x33333333], 2),
        ([-0.0, 0.0, 0.0], [1, 1, 1], [0, 0xFFFFFFFF, 0x5], 0),
        ([qnan("f32", 4), qnan("f32", 5), inf], [6, 6, 0], [1, 2, 3], 0),
    ],
    ("f32", MIN): [
        ([2.0, 2.0, 2.0], [7, 7, 7], [0xAAAAAAAA, 0xBBBBBBBB, 0xCCCCCCCC], 0),
        ([3.0, 2.0, 2.0], [0, 3, 3], [0x11111111, 0x22222222, 0x33333333], 1),
        ([-inf, 5.0, qnan("f32", 7)], [0, 1, 9], [4, 5, 6], 2),
    ],
    ("i64", MAX): [
        ([I64.min, I64.max, I64.max], [-5, -2, -9], None, 2),
        ([-1, 0, -1], [0, I64.min, I64.min], None, 1),
        ([I64.min, I64.min, I64.min], [I64.max, -3, -3], None, 1),
    ],
    ("i64", MIN): [
        ([I64.max, I64.min, I64.min], [0, -1, I64.min], None, 2),
        ([I64.max, I64.max, I64.max], [I64.min, I64.min, 0], None, 0),
        ([0, -1, 1], [0, 0, -1], None, 1),
    ],
}


def hand_inputs(dn, op):
    cases = HAND[(dn, op)]
    xs = []
    for r in range(3):
        pads = [c[2][r] for c in cases] if dn == "f32" else None
        xs.append(R.pairs(R.LOC[dn], [c[0][r] for c in cases], [c[1][r] for c in cases], pads))
    want = R.concat([xs[c[3]][i:i + 1] for i, c in enumerate(cases)])
    return xs, want


@pytest.mark.parametrize("key", sorted(HAND, key=str))
def test_restatement_and_oracle_match_the_hand_worked_cases(key):
    xs, want = hand_inputs(*key)
    got = R.allreduce_loc_np(xs, key[1])
    assert R.same(got, want), (key, got, want)
    assert R.same(LO.allreduce_loc(xs, key[1]), want), key


@pytest.mark.parametrize("op", [MAX, MIN])
@pytest.mark.parametrize("dn", ["f32", "f64", "i64"])
@pytest.mark.parametrize("n", range(1, 9))
def test_restatement_matches_the_oracle_on_tie_heavy_values(n, dn, op):
    xs = R.tie_heavy(dn, n, 4000, 100 * n + len(dn) + op)
    assert R.same(R.allreduce_loc_np(xs, op), LO.allreduce_loc(xs, op)), (n, dn, op)


@pytest.mark.parametrize("op", [MAX, MIN])
@pytest.mark.parametrize("dn", ["f32", "f64", "i64"])
@pytest.mark.parametrize("n", [2, 3, 5, 8])
def test_every_bracketing_gives_the_same_bytes(n, dn, op):
    """A left fold, a right fold and a pairwise tree agree byte for byte: whatever grid, unroll or
    world size a kernel combines in, the result is the same."""
    xs = R.tie_heavy(dn, n, 4000, 7000 + n)
    left = R.fold_left(xs, op)
    assert R.same(left, R.fold_right(xs, op)) and R.same(left, R.fold_tree(xs, op)), (n, dn, op)


@pytest.fixture(scope="module")
def loc_op_exe():
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-locop-"), "loc_op_test")
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "loc_op_test.cu"), "-cudart", "static"])
    return exe


def run_device_op(exe, xs, op):
    """OpMaxLoc / OpMinLoc (kernels.cuh) built for the host, folded over xs in three bracketings."""
    d = tempfile.mkdtemp(prefix="b200mpi-locop-run-")
    fin, fout = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
    R.concat(xs).tofile(fin)
    dt = xs[0].dtype
    out = subprocess.run([exe, str(mpi.api._LOC2DT[dt]), str(op), str(len(xs)), str(xs[0].size), fin, fout], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "loc op ok" in out.stdout, out.stdout + out.stderr
    return np.fromfile(fout, dtype=dt)


def test_device_op_matches_the_hand_worked_cases(loc_op_exe):
    for key in HAND:
        xs, want = hand_inputs(*key)
        assert R.same(run_device_op(loc_op_exe, xs, key[1]), want), key


@pytest.mark.parametrize("n", range(1, 9))
def test_device_op_matches_the_restatement(loc_op_exe, n):
    for dn in ("f32", "f64", "i64"):
        for op in (MAX, MIN):
            xs = R.tie_heavy(dn, n, 3000, 300 * n + op)
            assert R.same(run_device_op(loc_op_exe, xs, op), R.allreduce_loc_np(xs, op)), (n, dn, op)


class _Sized(mpi.Cuda):
    """A world of 3 seen from rank 1, without a library: every check below must fire before a call."""

    def Rank(self):
        return 1

    def Size(self):
        return 3


def test_pair_dtypes_are_the_c_layout():
    for dt, vt in ((mpi.LOC_F32, np.float32), (mpi.LOC_F64, np.float64), (mpi.LOC_I64, np.int64)):
        assert dt.itemsize == 16 and dt.fields["val"] == (np.dtype(vt), 0) and dt.fields["loc"] == (np.dtype(np.int64), 8)


def test_facade_checks_pairs_before_the_library():
    c = _Sized()
    a = np.zeros(4, mpi.LOC_F64)
    dev = mpi.DeviceSlice(4, mpi.LOC_F64, ptr=4096, owner=False)
    with pytest.raises(ValueError):
        c.AllreduceLoc(a, np.zeros(3, mpi.LOC_F64))               # lengths differ
    with pytest.raises(ValueError):
        c.AllreduceLoc(a, np.zeros(4, mpi.LOC_I64))               # pair types differ
    with pytest.raises(ValueError):
        c.AllreduceLoc(a, dev)                                    # memory kinds differ
    with pytest.raises(ValueError):
        c.ReduceLoc(dev, np.zeros(4, mpi.LOC_F64), MIN, 0)
    with pytest.raises(ValueError):
        c.AllreduceLoc(np.zeros(8, mpi.LOC_F32)[::2], np.zeros(4, mpi.LOC_F32))  # not contiguous
    for bad in (np.zeros(4, np.float64), np.zeros(4, np.dtype([("val", "<f4"), ("loc", "<i8")])), [1.0, 2.0], b"xy"):
        with pytest.raises(TypeError):                            # plain values, the packed 12-byte struct, other objects
            c.AllreduceLoc(bad, a)
        with pytest.raises(TypeError):
            c.ReduceLoc(bad, None, MAX, 0)


def test_other_calls_refuse_pairs():
    c = _Sized()
    a = np.zeros(4, mpi.LOC_F32)
    dev = mpi.DeviceSlice(4, mpi.LOC_I64, ptr=4096, owner=False)
    for x in (a, dev):
        for call in (lambda: c.Allreduce(x, x), lambda: c.Reduce(x, None), lambda: c.Bcast(x, 0), lambda: c.Send(x, 0, 1),
                     lambda: c.Isend(x, 0, 1), lambda: c.Receive(x, 0, 1), lambda: c.Allgather(x, x), lambda: c.Scan(x, x),
                     lambda: c.ReduceScatterv(x, x, [4, 0, 0])):
            with pytest.raises(TypeError):
                call()
    with pytest.raises(TypeError):
        mpi.DeviceSlice(4, np.dtype([("val", "<f4"), ("loc", "<i8")]), ptr=4096, owner=False)


def test_entries_before_init_report_not_initialised():
    lib = L.load()
    assert lib.b200mpi_size() == 0
    x = np.zeros(4, mpi.LOC_F64)
    assert lib.b200mpi_allreduce_loc(x.ctypes.data, x.ctypes.data, 4, L.F64, L.MAX, L.HOST) == L.ERR_NOT_INIT
    assert lib.b200mpi_reduce_loc(x.ctypes.data, None, 4, L.F64, L.MIN, 0, L.HOST) == L.ERR_NOT_INIT
    for call in (lambda: mpi.AllreduceLoc(x, x), lambda: mpi.ReduceLoc(x, x, mpi.MIN, 0)):
        with pytest.raises(mpi.MpiError) as e:
            call()
        assert e.value.code == L.ERR_NOT_INIT


def test_header_binding_and_library_carry_the_entries():
    lib = ctypes.CDLL(mpi.LIB_PATH)
    with open(os.path.join(ROOT, "include", "b200mpi.h")) as f:
        header = f.read()
    for name, decl in (("b200mpi_allreduce_loc", "int b200mpi_allreduce_loc(const void* send, void* recv, size_t count, int dtype, int op, int memkind);"),
                       ("b200mpi_reduce_loc", "int b200mpi_reduce_loc(const void* send, void* recv, size_t count, int dtype, int op, int root, int memkind);")):
        assert name in L.SYMBOLS and hasattr(lib, name) and decl in header
    assert L.load().b200mpi_version() == 200


@pytest.mark.parametrize("n", [1, 2])
def test_control_plane_world_refuses_the_loc_calls(n, monkeypatch):
    monkeypatch.setattr(_launch, "WORKER", LOC_WORKER)
    assert_world_ok(run_world(n, "loc_control_only", args=["--control-only"], timeout=120))


def test_cpp_facade_loc():
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-loc-"), "loc_facade_test")
    lib = os.path.join(ROOT, "mpi_b200", "lib")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "loc_facade_test.cpp"),
                           "-L" + lib, "-lb200mpi", "-Wl,-rpath," + lib, "-pthread"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "loc facade ok" in out.stdout, out.stdout + out.stderr
