"""One rank of a test world whose buffers lie past the 32-bit boundaries of the heap and of a message.
Usage as _worker.py: _large_worker.py <high|long> --out FILE [--parts ...] -mpi-* flags.

Scenario 'high': right after Init every rank allocates one arena that fills the heap from its start
(the first allocation lands at kHeapReserved) to ARENA_END, above 2^32, and every heap buffer of
_footprint_worker's calls is placed in it at a planned offset (PLACEMENT): rank 0's above 2^32, rank
1's send across 2^32 and its recv below, ranks 2 and 3 below at other offsets.  So the start-barrier
cells, the per-peer cells and the mailbox carry different high halves in one call, while the footprint
checks (guards, residues mod 16, the oracle in the order of the kernel that ran) apply unchanged.
Staging blocks of host views land above ARENA_END.

Scenario 'long': a world of two (or one) moves messages of 4 GiB and more, so byte positions pass
2^32 and element indices 2^31.  With two ranks every reduction is two-term, and a + b, max and min
of two values without NaN or a +0/-0 pair do not depend on the order, so the reference is plain:
f32 sums in f64 rounded once, f64 and i64 as the oracle's _apply (i64 wraps).  Inputs are generated
and every buffer (64 guard bytes on each side) is checked window by window (WINDOW bytes of the
generator stream), so host memory stays bounded."""
import argparse
import ctypes
import os
import sys
import time
import types
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _footprint_worker as F  # noqa: E402
import _rsv_worker as RW  # noqa: E402
import _scan_worker as SW  # noqa: E402
import _worker as W  # noqa: E402
from _worker import ALGOS, L, O, SEED, mpi  # noqa: E402

MiB, GiB = 1 << 20, 1 << 30
G32 = 1 << 32
RESERVED = 16 * MiB  # kHeapReserved: the control region before the first allocation
HIGH_HEAP = 4 * GiB + 512 * MiB
LONG_HEAP = 9 * GiB
ARENA_END = G32 + 256 * MiB
SLOT_BYTES = 64 * MiB
BIG_COUNT_BYTES = 4 * MiB  # the one long message of scenario 'high': rank 1's send crosses 2^32
V_BIG = (1 << 19) + 1  # elements rank 1 sends in the v-collectives of scenario 'high': over 256 KiB in u8
# heap offsets of each rank's buffer slots: the first buffer of a call takes slot 0, the next slot 1
PLACEMENT = ((G32 + 64 * MiB, G32 + 160 * MiB),  # rank 0: wholly above 2^32
             (G32 - 256 * 1024, 3 * GiB),         # rank 1: send straddles 2^32, recv below it
             (1 * GiB + 512, 2 * GiB + 1536),     # ranks 2 and 3: below, at other offsets
             (2 * GiB + 512 * MiB, 3 * GiB + 512 * MiB))
STAGE_BYTES = 8 * MiB  # the largest host view of scenario 'high' stays below pipe_min_bytes (8 MiB)
PROBE_BYTES = 512
WINDOW = 256 * MiB
THREADS = max(1, min(8, (os.cpu_count() or 2) // 2))  # window threads per rank of the world of two


def placement(n):
    """[(slot offsets of rank r)] for a world of n: the plan scenario 'high' follows."""
    return [PLACEMENT[r] for r in range(n)]


def symmetric_placement(n):
    """Every rank at rank 0's offsets: the multicast kernels need the same offset on every rank."""
    return [PLACEMENT[0]] * n


# ---- scenario 'high' ----------------------------------------------------------------------------
class Arena:
    """[RESERVED, ARENA_END) of this rank's heap, one allocation made right after Init."""

    def __init__(self, slots):
        self.mem = mpi.Alloc(ARENA_END - RESERVED, np.uint8)
        self.base = self.mem.ptr - RESERVED  # the heap's base: the arena is its first allocation
        self.slots = slots
        self.busy = set()
        self.placed = 0
        self.seen = {}

    def take(self, total):
        k = min(set(range(len(self.slots))) - self.busy)
        assert total <= SLOT_BYTES, "a buffer of %d bytes does not fit a slot" % total
        self.busy.add(k)
        return k, self.base + self.slots[k]

    def offset(self, ptr):
        return ptr - self.base


class Placed(F.Guarded):
    """F.Guarded whose heap allocation is the next free slot of the arena, at its planned offset."""
    arena = None

    def alloc(self, nbytes):
        A = Placed.arena
        self.slot, ptr = A.take(nbytes)
        lo, hi = ptr + self.head - A.base, ptr + self.head + self.nbody - A.base
        A.placed += 1
        side = "above" if lo >= G32 else "straddles" if hi > G32 else "below"
        A.seen[side] = A.seen.get(side, 0) + 1
        return mpi.DeviceSlice(nbytes, np.uint8, ptr, owner=False)

    def free(self):
        if self.kind == "heap":
            Placed.arena.busy.discard(self.slot)
        super().free()


def big_counts(dt, passes):
    """counts_for(..., 'edges') and one message of BIG_COUNT_BYTES + one element."""
    return F.counts_for(dt, passes, "edges") + [BIG_COUNT_BYTES // np.dtype(dt).itemsize + 1]


def part_reductions(R):
    n = R.n
    for algo in ("oneshot", "twoshot", "smem", "ring"):
        for di, dn in enumerate(("f32", "f64", "i64")):
            dt = F.DTYPES[dn]
            for ci, count in enumerate(big_counts(dt, F.allreduce_passes(algo, n, dt))):
                i = ci + di
                layout = F.LAYOUTS[i % 4]
                F.do_allreduce(R, algo, dn, count, layout, F.OPS[i % 3][0], layout in ("aligned", "mixed") and ci % 2 == 1,
                               R.kind_for(i, count * dt().itemsize))
    R.lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
    for di, dn in enumerate(("f32", "f64", "i64")):
        dt = F.DTYPES[dn]
        for ci, count in enumerate(big_counts(dt, F.allreduce_passes("twoshot", n, dt))):
            i = ci + di
            F.do_reduce(R, dn, count, F.LAYOUTS[i % 4], F.OPS[i % 3][0], 1 + i % (n - 1), ci % 2 == 1, R.kind_for(i, count * dt().itemsize))
        for ci, count in enumerate(big_counts(dt, [1024])):
            i = ci + di
            F.do_reduce_scatter(R, dn, count, F.LAYOUTS[(i + 1) % 4], F.OPS[i % 3][0], ci % 2 == 0, R.kind_for(i, count * n * dt().itemsize))
        for ci, count in enumerate(big_counts(dt, SW.scan_passes(n, dt))):
            i = ci + di
            for exclusive in (False, True):
                SW.do_footprint(R, dn, count, F.LAYOUTS[(i + exclusive) % 4], F.OPS[(i + exclusive) % 3][0], ci % 2 == 1,
                                R.kind_for(i + exclusive, count * dt().itemsize), exclusive)
        for ci, counts in enumerate(([3 + r for r in range(n)], [BIG_COUNT_BYTES // dt().itemsize + 1] + [5 * r for r in range(1, n)])):
            i = ci + di
            RW.do_footprint(R, dn, counts, F.LAYOUTS[i % 4], F.OPS[i % 3][0], ci == 0, R.kind_for(i, sum(counts) * dt().itemsize))
    R.lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
    R.lib.b200mpi_set_algo(L.COLL_REDUCE_SCATTER, 0)


def part_bytes(R):
    n = R.n
    for di, dn in enumerate(("u8", "f32", "i64")):
        dt = F.DTYPES[dn]
        es = dt().itemsize
        for algo in ("oneshot", "twoshot"):
            for ci, count in enumerate(big_counts(dt, [2047])):
                i = ci + di
                F.do_bcast(R, algo, dn, count, F.LAYOUTS[i % 4], (i + n // 2) % n, R.kind_for(i, count * es))
        R.lib.b200mpi_set_algo(L.COLL_BCAST, 0)
        for algo in ("oneshot", "ring"):
            for ci, count in enumerate(big_counts(dt, [2047])):
                i = ci + di
                F.do_allgather(R, algo, dn, count, F.LAYOUTS[i % 4], ci % 2 == 1, R.kind_for(i, count * n * es))
        R.lib.b200mpi_set_algo(L.COLL_ALLGATHER, 0)
        for ci, count in enumerate(big_counts(dt, [2047])):
            F.do_alltoall(R, dn, count, F.LAYOUTS[(ci + di) % 4], R.kind_for(ci + di, count * n * es))


def part_v(R):
    """F.part_v on tables in which rank 1 sends V_BIG elements, so that its send crosses 2^32."""
    n = R.n
    counts = [V_BIG if r == 1 else 5 + r for r in range(n)]
    skew = [[3 + i + 2 * j for j in range(n)] for i in range(n)]
    skew[1][0] = V_BIG
    F.part_v(R, counts, skew)


def part_p2p(R):
    """Send / Receive and Isend / Wait between ranks 2k and 2k+1, into the arenas."""
    F.part_p2p(R)
    rank, n = R.rank, R.n
    if rank >= n - n % 2:
        return
    dt = np.dtype(np.uint8)
    count = BIG_COUNT_BYTES + 3
    call = R.next_call("isend")
    x = F.gen_values(dt, 1, count, call)[0]
    what = "isend/wait u8 count=%d ranks %d->%d" % (count, rank & ~1, (rank & ~1) + 1)
    if rank % 2 == 0:
        send = Placed("heap", dt, count, 5, rank, call, body=x)
        mpi.Isend(send.view, rank ^ 1, 41)
        mpi.Wait(rank ^ 1, 41)
        F.check(send, what + " [send must be unchanged]")
        send.free()
    else:
        recv = Placed("heap", dt, count + 3, 11, rank, call)
        got = mpi.Receive(recv.view, rank ^ 1, 41)
        assert len(got) == count, "%s: received %d elements" % (what, len(got))
        recv.set_body(x)
        F.check(recv, what + " [recv: message, then 3 bytes that must not be written]")
        recv.free()


def part_nvls(R):
    F.part_nvls(R)


HIGH_PARTS = {"reductions": part_reductions, "bytes": part_bytes, "v": part_v, "p2p": part_p2p, "nvls": part_nvls}


def probe_staging(R):
    """One staged call (a host Allreduce), then a PROBE_BYTES allocation: first fit puts it in the
    lowest hole, so it lying above 2^32 shows that the staging blocks do too."""
    x = np.arange(1024, dtype=np.float32)
    y = np.zeros_like(x)
    mpi.Allreduce(x, y)
    assert np.array_equal(y, x * R.n), "staged probe allreduce"
    p = mpi.Alloc(PROBE_BYTES, np.uint8)
    off = Placed.arena.offset(p.ptr)
    p.free()
    assert off >= ARENA_END > G32, "rank %d: probe after the first staged call at heap offset %#x, below %#x" % (R.rank, off, ARENA_END)
    return off


def scenario_high(a):
    for m in (F, SW, RW):  # the footprint, scan and reduce-scatterv calls allocate through Placed
        m.Guarded = Placed
    slots = (symmetric_placement if a.parts == "nvls" else placement)(mpi.Size())[mpi.Rank()]
    Placed.arena = Arena(slots)
    R = F.Run(types.SimpleNamespace(trim="edges"))
    A = Placed.arena
    probe = probe_staging(R)
    secs = {}
    for name in a.parts.split(","):
        t0 = time.time()
        HIGH_PARTS[name](R)
        mpi.Barrier()
        secs[name] = round(time.time() - t0, 2)
    A.mem.free()
    return {"checked": R.call, "by_part": R.done, "seconds": secs, "nvls": R.nvls, "skipped": sorted(R.skipped),
            "slots": ["%#x" % s for s in slots], "probe": "%#x" % probe, "placed": A.placed, "sides": A.seen}


# ---- scenario 'long' ----------------------------------------------------------------------------
def window(dn, seed, lo, hi):
    """Elements [lo, hi) of a long input: oracle.fill_at's stream of `seed`, floats negated where
    i % 3 == 1 (the sign depends on the position only, so two ranks never hold +0 and -0 at one
    position); u8 the low byte of the i64 stream."""
    if dn == "u8":
        return O.fill_at(np.int64, seed, lo, hi - lo).astype(np.uint8)
    x = O.fill_at(F.DTYPES[dn], seed, lo, hi - lo)
    if dn != "i64":
        s = (1 - lo) % 3
        x[s::3] = -x[s::3]
    return x


def windows(count, dt):
    """[lo, hi) element ranges of at most WINDOW bytes of the generator stream (8 bytes per element)."""
    step = WINDOW // 8
    return [(lo, min(lo + step, count)) for lo in range(0, count, step)]


def reduce2(dn, op, a, b):
    """The two-term reduction, the oracle's _apply: an f32 sum is float32(float64(a) + float64(b)),
    exact and then rounded once, which f32 addition gives directly (test_large_cpu checks it)."""
    with np.errstate(over="ignore", invalid="ignore"):
        return O._apply(op, a, b)


def splice(at, first, second):
    """A generator that is `first` below element `at` and `second(lo - at, hi - at)` from it on."""
    def gen(lo, hi):
        parts = []
        if lo < at:
            parts.append(first(lo, min(hi, at)))
        if hi > at:
            parts.append(second(max(lo, at) - at, hi - at))
        return np.concatenate(parts)
    return gen


def shifted(gen, by):
    return lambda lo, hi: gen(lo + by, hi + by)


class Long:
    """`count` elements at byte `off` past a GUARD-byte head guard of one allocation: the heap, pinned
    host memory from b200mpi_host_alloc, or a pageable numpy array.  fill and check run the windows on
    THREADS threads (the generator, numpy and the copies release the GIL)."""
    live = 0  # heap bytes this rank's Long buffers hold now, and the most they held at once
    peak = 0

    def __init__(self, dn, count, off, tag, kind="heap"):
        self.kind, self.dn, self.dt, self.count = kind, dn, np.dtype(F.DTYPES[dn]), int(count)
        self.head = F.GUARD + off
        self.nbody = self.count * self.dt.itemsize
        self.total = self.head + self.nbody + F.GUARD
        rank = mpi.Rank()
        self.guards = F.guard_pattern(rank, tag, self.head), F.guard_pattern(rank, tag + 1, F.GUARD)
        self.hp = None
        if kind == "heap":
            self.mem = mpi.Alloc(self.total, np.uint8)
            self.ptr = self.mem.ptr
            Long.live += -(-self.total // 512) * 512
            Long.peak = max(Long.peak, Long.live)
        else:
            if kind == "pinned":
                raw, self.hp = W.pinned_array(self.total + 64, np.uint8)
            else:
                raw = np.empty(self.total + 64, dtype=np.uint8)
            s = (-raw.ctypes.data) % 64
            self.mem = raw[s:s + self.total]
            self.ptr = self.mem.ctypes.data
        self._put_bytes(0, self.guards[0])
        self._put_bytes(self.head + self.nbody, self.guards[1])

    def _put_bytes(self, at, b):
        if self.kind == "heap":
            mpi.DeviceSlice(b.size, np.uint8, self.ptr + at, owner=False).copy_from_host(b)
        else:
            self.mem[at:at + b.size] = b

    def _get_bytes(self, at, k):
        if self.kind == "heap":
            return mpi.DeviceSlice(k, np.uint8, self.ptr + at, owner=False).to_host()
        return np.array(self.mem[at:at + k], copy=True)

    def view(self):
        if self.kind == "heap":
            return mpi.DeviceSlice(self.count, self.dt, self.ptr + self.head, owner=False)
        return self.mem[self.head:self.head + self.nbody].view(self.dt)

    def fill(self, gen):
        es = self.dt.itemsize
        put = lambda w: self._put_bytes(self.head + w[0] * es, np.ascontiguousarray(gen(*w), dtype=self.dt).view(np.uint8))  # noqa: E731
        with ThreadPoolExecutor(THREADS) as ex:
            list(ex.map(put, windows(self.count, self.dt)))

    def check(self, gen, what):
        """Both guards and every element against gen, window by window; the first difference is
        reported with its element index and its byte position in the message."""
        es = self.dt.itemsize
        for name, at, want in (("head guard", 0, self.guards[0]), ("tail guard", self.head + self.nbody, self.guards[1])):
            got = self._get_bytes(at, want.size)
            bad = np.flatnonzero(got != want)
            if bad.size:
                raise AssertionError("%s: %s byte %d written: got 0x%02x want 0x%02x" % (what, name, bad[0], got[bad[0]], want[bad[0]]))

        def one(w):
            lo, hi = w
            got = self._get_bytes(self.head + lo * es, (hi - lo) * es).view(self.dt)
            want = np.ascontiguousarray(gen(lo, hi), dtype=self.dt)
            bad = np.flatnonzero(got.view(np.uint8) != want.view(np.uint8))
            if not bad.size:
                return None
            i = lo + int(bad[0]) // es
            return "%s: element %d (byte %d of the message) got %r want %r (%d bytes differ in [%d, %d))" % (
                what, i, i * es, got[i - lo], want[i - lo], bad.size, lo, hi)
        with ThreadPoolExecutor(THREADS) as ex:
            errors = [e for e in ex.map(one, windows(self.count, self.dt)) if e]
        if errors:
            raise AssertionError(errors[0])

    def free(self):
        if self.kind == "heap":
            self.mem.free()
            Long.live -= -(-self.total // 512) * 512
        elif self.hp is not None:
            L.load().b200mpi_host_free(self.hp)
            self.hp = None
        self.mem = None


class LongRun:
    def __init__(self):
        self.lib = L.load()
        self.rank, self.n = mpi.Rank(), mpi.Size()
        self.call = 0
        self.done = []
        self.heap_peak = 0

    def next(self, what):
        self.call += 1
        self.done.append(what)
        W.trace(what)
        return self.call

    def seed(self, call, r):
        return SEED + 7919 * call + r

    def gen(self, dn, call, r):
        """Rank r's input of `call`."""
        return lambda lo, hi: window(dn, self.seed(call, r), lo, hi)

    def used(self):
        """Note the heap bytes in use now (buffers and staging blocks): the most is reported."""
        used = ctypes.c_size_t()
        self.lib.b200mpi_heap_info(None, ctypes.byref(used), None)
        self.heap_peak = max(self.heap_peak, used.value)


def reduced(dn, op, ins, shift=0):
    """The two-rank reduction of ins, from element `shift` of each input on."""
    return lambda lo, hi: reduce2(dn, op, ins[0](lo + shift, hi + shift), ins[1](lo + shift, hi + shift))


def long_reduce(R, algo, dn, opname, count, inplace, root=None):
    """Allreduce (root None) or Reduce of two ranks' `count` elements, the views 16-byte aligned so
    that the vector bodies run; a Reduce leaves the non-root recv unwritten."""
    rank = R.rank
    op, oop = {o[0]: (o[1], o[2]) for o in F.OPS}[opname]
    coll = "allreduce" if root is None else "reduce root=%d" % root
    call = R.next("%s %s %s %s count=%d inplace=%s" % (coll, algo, dn, opname, count, inplace))
    what = R.done[-1] + " rank=%d" % rank
    ins = [R.gen(dn, call, r) for r in range(2)]
    send = Long(dn, count, 0, call)
    send.fill(ins[rank])
    recv = send if inplace else Long(dn, count, 16, call + 2)
    before = R.gen(dn, call, 9)
    if not inplace:
        recv.fill(before)
    R.lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS[algo])
    if root is None:
        mpi.Allreduce(send.view(), recv.view(), op)
    else:
        mpi.Reduce(send.view(), recv.view(), op, root)
    R.lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
    R.used()
    if root is None or rank == root:
        recv.check(reduced(dn, oop, ins), what + " [recv]")
    else:
        recv.check(before, what + " [non-root recv must not be written]")
    if not inplace:
        send.check(ins[rank], what + " [send must be unchanged]")
        recv.free()
    send.free()


def part_long_allreduce(R):
    """f32 SUM in place at 2^31 + 5 elements (element indices and the last rank's tail past 2^31) with
    the two-shot, TMA two-shot and ring kernels; f64 MAX out of place at 2^29 + 3 (4 GiB + 24 bytes),
    two-shot and ring, and a Reduce to root 1."""
    for algo in ("twoshot", "smem", "ring"):
        long_reduce(R, algo, "f32", "sum", (1 << 31) + 5, True)
    for algo in ("twoshot", "ring"):
        long_reduce(R, algo, "f64", "max", (1 << 29) + 3, False)
    long_reduce(R, "twoshot", "f64", "max", (1 << 29) + 3, False, root=1)


def part_long_reduce(R):
    """i64 SUM ReduceScatter of 2^28 + 1 elements per block; f32 SUM Scan in place at 2^30 + 5 and i64
    MIN Exscan at 2^29 + 3; f32 SUM ReduceScatterv with table [2^30 + 3, 7], whose second block starts
    at byte 4 GiB + 12 of every send, past 2^32 and not 16-byte aligned."""
    rank = R.rank
    count = (1 << 28) + 1
    call = R.next("reduce_scatter i64 sum count=%d" % count)
    what = R.done[-1] + " rank=%d" % rank
    ins = [R.gen("i64", call, r) for r in range(2)]
    send, recv = Long("i64", 2 * count, 0, call), Long("i64", count, 16, call + 2)
    send.fill(ins[rank])
    mpi.ReduceScatter(send.view(), recv.view(), mpi.SUM)
    R.used()
    recv.check(reduced("i64", O.SUM, ins, rank * count), what + " [recv]")
    send.check(ins[rank], what + " [send must be unchanged]")
    send.free()
    recv.free()
    for dn, opname, count, exclusive in (("f32", "sum", (1 << 30) + 5, False), ("i64", "min", (1 << 29) + 3, True)):
        op, oop = {o[0]: (o[1], o[2]) for o in F.OPS}[opname]
        call = R.next("%s %s %s count=%d" % ("exscan" if exclusive else "scan", dn, opname, count))
        what = R.done[-1] + " rank=%d" % rank
        ins = [R.gen(dn, call, r) for r in range(2)]
        send = Long(dn, count, 0, call)
        send.fill(ins[rank])
        recv = Long(dn, count, 16, call + 2) if exclusive else send
        before = R.gen(dn, call, 9)
        if exclusive:
            recv.fill(before)
        (mpi.Exscan if exclusive else mpi.Scan)(send.view(), recv.view(), op)
        R.used()
        if exclusive:
            recv.check(before if rank == 0 else ins[0], what + " [recv]")
            send.check(ins[rank], what + " [send must be unchanged]")
            recv.free()
        else:
            recv.check(ins[0] if rank == 0 else reduced(dn, oop, ins), what + " [recv]")
        send.free()
    counts = [(1 << 30) + 3, 7]
    call = R.next("reduce_scatterv f32 sum table=%s" % counts)
    what = R.done[-1] + " rank=%d" % rank
    ins = [R.gen("f32", call, r) for r in range(2)]
    send, recv = Long("f32", sum(counts), 0, call), Long("f32", counts[rank], 4, call + 2)
    send.fill(ins[rank])
    mpi.ReduceScatterv(send.view(), recv.view(), counts, mpi.SUM)
    R.used()
    recv.check(reduced("f32", O.SUM, ins, rank * counts[0]), what + " [recv]")
    send.check(ins[rank], what + " [send must be unchanged]")
    send.free()
    recv.free()


def part_long_bytes(R):
    """u8 Bcast of 2^32 + 7 bytes from root 1 with both P2P algorithms; push and ring Allgather of
    2^31 + 3 bytes per rank; Alltoall with blocks of 2^31 + 1 bytes."""
    rank = R.rank
    count = (1 << 32) + 7
    for algo in ("oneshot", "twoshot"):
        call = R.next("bcast u8 %s count=%d root=1" % (algo, count))
        buf = Long("u8", count, 3, call)
        buf.fill(R.gen("u8", call, rank))
        R.lib.b200mpi_set_algo(L.COLL_BCAST, ALGOS[algo])
        mpi.Bcast(buf.view(), 1)
        R.lib.b200mpi_set_algo(L.COLL_BCAST, 0)
        R.used()
        buf.check(R.gen("u8", call, 1), R.done[-1] + " rank=%d" % rank)
        buf.free()
    count = (1 << 31) + 3
    for algo in ("oneshot", "ring"):
        call = R.next("allgather u8 %s count=%d" % (algo, count))
        what = R.done[-1] + " rank=%d" % rank
        send, recv = Long("u8", count, 1, call), Long("u8", 2 * count, 9, call + 2)
        send.fill(R.gen("u8", call, rank))
        R.lib.b200mpi_set_algo(L.COLL_ALLGATHER, ALGOS[algo])
        mpi.Allgather(send.view(), recv.view())
        R.lib.b200mpi_set_algo(L.COLL_ALLGATHER, 0)
        R.used()
        recv.check(splice(count, R.gen("u8", call, 0), R.gen("u8", call, 1)), what + " [recv]")
        send.check(R.gen("u8", call, rank), what + " [send must be unchanged]")
        send.free()
        recv.free()
    count = (1 << 31) + 1
    call = R.next("alltoall u8 count=%d" % count)
    what = R.done[-1] + " rank=%d" % rank
    send, recv = Long("u8", 2 * count, 7, call), Long("u8", 2 * count, 2, call + 2)
    send.fill(R.gen("u8", call, rank))
    mpi.Alltoall(send.view(), recv.view())
    R.used()
    recv.check(splice(count, shifted(R.gen("u8", call, 0), rank * count), shifted(R.gen("u8", call, 1), rank * count)), what + " [recv]")
    send.check(R.gen("u8", call, rank), what + " [send must be unchanged]")
    send.free()
    recv.free()


def part_long_v(R):
    """u8 Gatherv to root 0 and Scatterv from root 1 with table [2^32 + 5, 3], Allgatherv with
    [3, 2^32 + 5], and Alltoallv with one block of 2^32 + 1 bytes."""
    rank = R.rank
    u8 = lambda call, r: R.gen("u8", call, r)  # noqa: E731
    big = (1 << 32) + 5
    counts = [big, 3]
    call = R.next("gatherv u8 root=0 counts=%s" % counts)
    what = R.done[-1] + " rank=%d" % rank
    send = Long("u8", counts[rank], 5, call)
    send.fill(u8(call, rank))
    recv = Long("u8", sum(counts), 0, call + 2) if rank == 0 else None
    mpi.Gatherv(send.view(), recv.view() if recv else None, 0, counts)
    R.used()
    if recv:
        recv.check(splice(big, u8(call, 0), u8(call, 1)), what + " [root recv]")
        recv.free()
    send.check(u8(call, rank), what + " [send must be unchanged]")
    send.free()
    call = R.next("scatterv u8 root=1 counts=%s" % counts)
    what = R.done[-1] + " rank=%d" % rank
    send = Long("u8", sum(counts), 6, call) if rank == 1 else None
    if send:
        send.fill(u8(call, 1))
    recv = Long("u8", counts[rank], 13, call + 2)
    mpi.Scatterv(send.view() if send else None, recv.view(), counts, 1)
    R.used()
    recv.check(shifted(u8(call, 1), 0 if rank == 0 else big), what + " [recv]")
    if send:
        send.check(u8(call, 1), what + " [root send must be unchanged]")
        send.free()
    recv.free()
    counts = [3, big]
    call = R.next("allgatherv u8 counts=%s" % counts)
    what = R.done[-1] + " rank=%d" % rank
    send, recv = Long("u8", counts[rank], 1, call), Long("u8", sum(counts), 11, call + 2)
    send.fill(u8(call, rank))
    mpi.Allgatherv(send.view(), recv.view(), counts)
    R.used()
    recv.check(splice(3, u8(call, 0), u8(call, 1)), what + " [recv]")
    send.check(u8(call, rank), what + " [send must be unchanged]")
    send.free()
    recv.free()
    table = [[3, (1 << 32) + 1], [5, 7]]  # table[i][j]: elements rank i sends to rank j
    row, col = table[rank], [table[0][rank], table[1][rank]]
    call = R.next("alltoallv u8 table=%s" % table)
    what = R.done[-1] + " rank=%d" % rank
    send, recv = Long("u8", sum(row), 4, call), Long("u8", sum(col), 8, call + 2)
    send.fill(u8(call, rank))
    mpi.Alltoallv(send.view(), row, recv.view(), col)
    R.used()
    at = [sum(table[r][:rank]) for r in range(2)]  # where rank r's block for this rank starts in its send
    recv.check(splice(col[0], shifted(u8(call, 0), at[0]), shifted(u8(call, 1), at[1])), what + " [recv]")
    send.check(u8(call, rank), what + " [send must be unchanged]")
    send.free()
    recv.free()


def part_long_p2p(R):
    """Send / Receive of 2^32 + 3 bytes from heap memory (a direct post), from a pageable numpy array
    (the staging ring) and through Isend / Wait (staged whole), each into a heap buffer 13 bytes
    longer that must report the length and leave the rest unwritten."""
    rank = R.rank
    count = (1 << 32) + 3
    for how in ("heap", "pageable", "isend"):
        call = R.next("p2p %s u8 count=%d 0->1" % (how, count))
        what = R.done[-1] + " rank=%d" % rank
        msg = R.gen("u8", call, 0)
        if rank == 0:
            send = Long("u8", count, 3, call, kind="heap" if how == "heap" else "pageable")
            send.fill(msg)
            if how == "isend":
                mpi.Isend(send.view(), 1, 50)
                R.used()
                mpi.Wait(1, 50)
            else:
                mpi.Send(send.view(), 1, 50)
            send.check(msg, what + " [send must be unchanged]")
            send.free()
        else:
            recv = Long("u8", count + 13, 6, call + 2)
            before = R.gen("u8", call, 9)
            recv.fill(before)
            got = mpi.Receive(recv.view(), 0, 50)
            R.used()
            assert len(got) == count, "%s: Receive reported %d bytes" % (what, len(got))
            recv.check(splice(count, msg, shifted(before, count)), what + " [recv: message, then 13 bytes that must not be written]")
            recv.free()


def part_long_hostpipe(R):
    """The chunked host-slice pipeline: an in-place f32 SUM Allreduce of 2^30 + 5 elements from pinned
    and from pageable memory, about a thousand chunk launches each."""
    rank = R.rank
    count = (1 << 30) + 5
    for kind in ("pinned", "pageable"):
        call = R.next("host-slice allreduce f32 sum %s count=%d" % (kind, count))
        ins = [R.gen("f32", call, r) for r in range(2)]
        buf = Long("f32", count, 4 * rank, call, kind=kind)
        buf.fill(ins[rank])
        launches = R.lib.b200mpi_launch_count()
        mpi.Allreduce(buf.view(), buf.view(), mpi.SUM)
        launches = R.lib.b200mpi_launch_count() - launches
        R.used()
        R.done[-1] += " (%d launches)" % launches
        buf.check(reduced("f32", O.SUM, ins), R.done[-1] + " rank=%d" % rank)
        chunks = count * 4 // L.get_param("pipe_chunk_bytes")
        assert launches >= chunks, "%s: fewer launches than %d-byte pipeline chunks (%d)" % (R.done[-1], L.get_param("pipe_chunk_bytes"), chunks)
        buf.free()


def part_long_local(R):
    """World of one: an out-of-place f32 Allreduce of 4 GiB + 20 bytes is a local copy:
    copy_local_kernel when send and recv agree mod 16, copy_bytes_kernel when they do not."""
    count = (1 << 30) + 5
    for soff, roff in ((0, 0), (0, 4)):
        call = R.next("world of one allreduce f32 count=%d offsets(send,recv)=(%d,%d)" % (count, soff, roff))
        x = R.gen("f32", call, 0)
        send, recv = Long("f32", count, soff, call), Long("f32", count, roff, call + 2)
        send.fill(x)
        mpi.Allreduce(send.view(), recv.view(), mpi.SUM)
        R.used()
        recv.check(x, R.done[-1] + " [recv]")
        send.check(x, R.done[-1] + " [send must be unchanged]")
        send.free()
        recv.free()


LONG_PARTS = {"allreduce": part_long_allreduce, "reduce": part_long_reduce, "bytes": part_long_bytes, "v": part_long_v,
              "p2p": part_long_p2p, "hostpipe": part_long_hostpipe, "local": part_long_local}


def scenario_long(a):
    R = LongRun()
    secs = {}
    for name in a.parts.split(","):
        t0 = time.time()
        LONG_PARTS[name](R)
        mpi.Barrier()
        secs[name] = round(time.time() - t0, 2)
    return {"checked": R.call, "calls": R.done, "seconds": secs, "heap_peak": R.heap_peak, "buffer_peak": Long.peak}


if __name__ == "__main__":
    ap = argparse.ArgumentParser(add_help=False)
    ap.add_argument("--parts", required=True)
    opts, rest = ap.parse_known_args(sys.argv[1:])
    sys.argv = [sys.argv[0]] + rest  # _worker.main parses the rest
    W.SCENARIOS["high"] = lambda a: scenario_high(opts)
    W.SCENARIOS["long"] = lambda a: scenario_long(opts)
    W.main()
