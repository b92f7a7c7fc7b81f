"""The plans of test_gpu_large.py without a GPU: where _large_worker.py places its buffers, replayed
against a host build of the heap's sub-allocator; the windowed input generator against the oracle's
whole streams, past 2^31 and 2^32 included; and the plain two-rank reference against the oracle in
every order the kernels use."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import _footprint_worker as F
import _large_worker as LW
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G32 = 1 << 32


@pytest.fixture(scope="module")
def heap():
    """A function that sends allocator commands to a host build of heap.cpp and returns its replies."""
    exe = os.path.join(tempfile.mkdtemp(prefix="b200mpi-heap-plan-"), "heap_plan")
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-std=c++17", "-O1", "-o", exe, os.path.join(ROOT, "tests", "cpp", "heap_plan.cpp"),
                           os.path.join(ROOT, "mpi_b200", "csrc", "heap.cpp"), os.path.join(ROOT, "mpi_b200", "csrc", "ctrl.cpp"), "-cudart", "static", "-lpthread"])

    def run(cmds):
        out = subprocess.run([exe], input="\n".join(cmds) + "\n", capture_output=True, text=True, timeout=60)
        assert out.returncode == 0, out.stderr
        return out.stdout.split()
    return run


def max_buffer(n):
    """The largest allocation a Placed buffer of scenario 'high' asks for: the 4 MiB message of
    every collective (Allgather and Alltoall recv n of them), with guards and the largest offset."""
    return max(F.zones(LW.BIG_COUNT_BYTES // es + 1, dt, 15 + 32)[3] * n for es, dt in ((1, np.uint8), (4, np.float32), (8, np.int64)))


@pytest.mark.parametrize("n", [2, 3, 4])
def test_high_offset_plan_lands_where_planned(heap, n):
    """In the heap of scenario 'high' the arena is the first allocation (at kHeapReserved) and ends
    at ARENA_END; every slot lies inside it, slots of a rank do not overlap, rank 0's lie above 2^32,
    rank 1's first crosses 2^32 with the long message and its second lies below; then the staging
    blocks of host views and the probe land above 2^32, and all of it fits the heap."""
    arena = LW.ARENA_END - LW.RESERVED
    replies = heap(["reset %d" % LW.HIGH_HEAP, "alloc %d" % arena,
                    "alloc %d" % LW.STAGE_BYTES, "alloc %d" % (LW.STAGE_BYTES * n), "alloc %d" % LW.PROBE_BYTES, "used"])
    assert replies[0] == "ok"
    first, st0, st1, probe, used = replies[1:]
    assert first != "nomem" and int(first) == LW.RESERVED, "the arena is not the first allocation at kHeapReserved: %s" % first
    for what, off in (("send staging", st0), ("recv staging", st1), ("probe", probe)):
        assert off != "nomem", "%s does not fit a heap of %d bytes after the arena" % (what, LW.HIGH_HEAP)
        assert int(off) >= LW.ARENA_END > G32, "%s at heap offset %#x lies below 2^32" % (what, int(off))
    assert int(used) + LW.RESERVED <= LW.HIGH_HEAP
    big = max_buffer(n)
    assert big <= LW.SLOT_BYTES, (big, LW.SLOT_BYTES)
    for r, slots in enumerate(LW.placement(n)):
        for k, s in enumerate(slots):
            assert s % 512 == 0, "rank %d slot %d at heap offset %#x is not 512-byte aligned" % (r, k, s)
            assert LW.RESERVED <= s and s + LW.SLOT_BYTES <= LW.ARENA_END, "rank %d slot %d at heap offset %#x leaves the arena" % (r, k, s)
        for a in range(len(slots)):
            for b in range(a + 1, len(slots)):
                assert slots[a] + LW.SLOT_BYTES <= slots[b] or slots[b] + LW.SLOT_BYTES <= slots[a], "rank %d slots %d and %d overlap" % (r, a, b)
        if r == 0:
            assert all(s >= G32 for s in slots), "rank 0 slot at heap offset %#x lies below 2^32" % min(slots)
        if r == 1:
            lo = slots[0] + F.GUARD
            assert lo < G32 < lo + LW.BIG_COUNT_BYTES, "rank 1 send at heap offset %#x does not cross 2^32" % slots[0]
            assert slots[1] + LW.SLOT_BYTES <= G32, "rank 1 recv at heap offset %#x does not lie below 2^32" % slots[1]
        if r >= 2:
            assert all(s + LW.SLOT_BYTES <= G32 for s in slots), "rank %d slot at heap offset %#x does not lie below 2^32" % (r, max(slots))
    # the cells of one call carry different high halves
    highs = {s >> 32 for slots in LW.placement(n) for s in slots}
    assert highs == {0, 1}, highs
    assert all(s >= G32 for s in LW.symmetric_placement(n)[0]) and len(set(LW.symmetric_placement(n))) == 1


@pytest.mark.parametrize("dn", ["u8", "f32", "f64", "i64"])
def test_windows_concatenate_to_the_whole_stream(dn, monkeypatch):
    """At a small window size the windows of the generator cover the buffer exactly once and
    concatenate to oracle.fill's stream (signs by position for floats, the low byte for u8)."""
    monkeypatch.setattr(LW, "WINDOW", 8 * 97)  # 97 elements per window: windows end off any vector boundary
    count = 1000
    seed = LW.SEED + 5
    ws = LW.windows(count, None)
    assert ws[0][0] == 0 and ws[-1][1] == count and all(a[1] == b[0] for a, b in zip(ws, ws[1:]))
    got = np.concatenate([LW.window(dn, seed, lo, hi) for lo, hi in ws])
    if dn == "u8":
        want = O.fill(np.int64, seed, count).astype(np.uint8)
    else:
        want = O.fill(F.DTYPES[dn], seed, count)
        if dn != "i64":
            want[1::3] = -want[1::3]
    assert got.dtype == np.dtype(F.DTYPES[dn]) and np.array_equal(got.view(np.uint8), want.view(np.uint8))


@pytest.mark.parametrize("dn", ["u8", "f32", "f64", "i64"])
@pytest.mark.parametrize("start", [(1 << 31) - 3, G32 - 5, G32 + 7, (9 << 30) - 16])
def test_windows_past_the_32_bit_boundaries_follow_splitmix(dn, start):
    """Windows that start near and past 2^31 and 2^32 equal the generator restated element by element
    from oracle_splitmix64: fill_at keeps the 64-bit position in every element."""
    seed = LW.SEED + 11
    got = LW.window(dn, seed, start, start + 24)
    for k in range(24):
        i = start + k
        z = O.lib().oracle_splitmix64(seed, i)
        if dn in ("u8", "i64"):
            want = np.array([z & 0xFF if dn == "u8" else z], dtype=np.uint64).astype(np.int64 if dn == "i64" else np.uint8)[0]
        elif dn == "f32":
            want = np.float32(z >> 40) * np.float32(1.0 / 16777216.0)
        else:
            want = np.float64(z >> 11) * (1.0 / 9007199254740992.0)
        if dn in ("f32", "f64") and i % 3 == 1:
            want = -want
        assert got[k].tobytes() == np.asarray(want, dtype=got.dtype).tobytes(), \
            "%s window at %d: element %d (byte %d) got %r want %r" % (dn, start, i, i * got.dtype.itemsize, got[k], want)


def two_rank_inputs(dn):
    """Two ranks' inputs with every pairing of signed zeros, infinities, extremes and plain values."""
    dt = np.dtype(F.DTYPES[dn])
    if dn == "i64":
        pool = np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, -1, 0, 1, 12345, -98765], dtype=dt)
    else:
        fi = np.finfo(dt)
        pool = np.array([0.0, -0.0, np.inf, -np.inf, fi.max, -fi.max, fi.tiny, fi.smallest_subnormal, -fi.smallest_subnormal,
                         1.0, -1.0, 1.0 + fi.eps, 3.0, -2.5e-3], dtype=dt)
    a, b = np.meshgrid(pool, pool)
    x0, x1 = a.reshape(-1), b.reshape(-1)
    plain = [LW.window(dn, LW.SEED + r, 0, 4096) for r in range(2)]
    return [np.concatenate([x0, plain[0]]), np.concatenate([x1, plain[1]])]


def signed_zero_pairs(xs):
    return (xs[0] == 0) & (xs[1] == 0) & (np.signbit(xs[0]) != np.signbit(xs[1]))


@pytest.mark.parametrize("dn", ["f32", "f64", "i64"])
@pytest.mark.parametrize("opname", ["sum", "max", "min"])
def test_two_rank_reference_equals_the_oracle_in_every_order(dn, opname):
    """For two ranks the plain reference equals oracle_allreduce in rank, tree and ring order, bit for
    bit: a + b is b + a, and max and min of two values are order-free too, except where one rank
    holds +0 and the other -0 (b > a ? b : a keeps the first operand).  The long-message inputs
    never pair those, since their sign depends on the position only."""
    op = {o[0]: o[2] for o in F.OPS}[opname]
    xs = two_rank_inputs(dn)
    ref = LW.reduce2(dn, op, xs[0], xs[1])
    zeros = signed_zero_pairs(xs)
    assert dn == "i64" or zeros.any(), "the inputs must pair +0 with -0"
    for order in (O.ORDER_RANK, O.ORDER_TREE, O.ORDER_RING):
        got = O.allreduce(xs, op=op, order=order)
        same = got.view(np.uint8).reshape(got.size, -1) == ref.view(np.uint8).reshape(ref.size, -1)
        same = same.all(axis=1)
        if op != O.SUM:
            # +0 against -0 is where MAX / MIN depend on the order; NaN-free elsewhere
            assert same[~zeros].all(), "%s %s order %d differs at %s" % (dn, opname, order, np.flatnonzero(~same & ~zeros)[:5])
        else:
            assert same.all(), "%s sum order %d differs at %s" % (dn, order, np.flatnonzero(~same)[:5])
    if op != O.SUM and dn != "i64":
        rank_order = O.allreduce(xs, op=op, order=O.ORDER_RANK)
        swapped = O.allreduce(xs[::-1], op=op, order=O.ORDER_RANK)
        assert not np.array_equal(rank_order[zeros].view(np.uint8), swapped[zeros].view(np.uint8)), \
            "+0 against -0 was expected to depend on the order of %s" % opname


@pytest.mark.parametrize("dn", ["f32", "f64"])
def test_long_inputs_never_pair_signed_zeros(dn):
    """The sign rule gives both ranks the same sign at every position, so the long-message MAX / MIN
    references hold in every order even where both values are zero."""
    for lo in (0, (1 << 31) - 7, G32 + 1):
        xs = [LW.window(dn, LW.SEED + 3 * r + 1, lo, lo + 3000) for r in range(2)]
        assert np.array_equal(np.signbit(xs[0]), np.signbit(xs[1]))


def test_f32_sum_reference_is_rounded_once():
    """float32(float64(a) + float64(b)) is the correctly rounded f32 sum, which is what f32 addition
    gives in either order."""
    xs = [LW.window("f32", LW.SEED + r, 0, 1 << 16) for r in range(2)]
    ref = (xs[0].astype(np.float64) + xs[1].astype(np.float64)).astype(np.float32)
    assert np.array_equal(LW.reduce2("f32", O.SUM, xs[0], xs[1]), ref) and np.array_equal(LW.reduce2("f32", O.SUM, xs[1], xs[0]), ref)
    assert not np.array_equal(ref.astype(np.float64), xs[0].astype(np.float64) + xs[1].astype(np.float64)), "no sum was rounded"
