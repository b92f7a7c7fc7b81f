"""One rank of a test world for Send, Isend, Wait and Receive.
Usage as _worker.py: _p2p_worker.py p2p --out FILE --parts matrix,self,errors,depth -mpi-* flags.

Every message is a guarded buffer (_kinds_worker.Buf: heap, torch, pinned, torch pinned or pageable
memory, 16-byte aligned or not) holding the footprint test's values, and every receive has room for 3
more elements than arrive, which must stay unwritten; the send buffer must come back unchanged.  Where
one rank runs one call at a time, each call must also leave this rank's heap as it found it (after Wait,
for an Isend) and launch exactly the kernels _p2p_plan.py predicts for its side, which shows that the
planned sender and receiver layouts are the ones that ran."""
import argparse
import ctypes
import os
import random
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _footprint_worker as F  # noqa: E402
import _p2p_plan as P  # noqa: E402
import _worker as W  # noqa: E402
from _kinds_worker import MISALIGN, Buf  # noqa: E402
from _worker import L, O, mpi  # noqa: E402

DT = {k: np.dtype(v) for k, v in F.DTYPES.items()}
CODE = {k: O.NP2DT[v] for k, v in DT.items()}


class Run:
    def __init__(self):
        self.lib = L.load()
        self.rank, self.n = mpi.Rank(), mpi.Size()
        self.call = 0
        self.pairs = {}
        self.done = {}

    def next_call(self, part):
        self.call += 1
        self.done[part] = self.done.get(part, 0) + 1
        return self.call

    def set(self, name, v):
        assert self.lib.b200mpi_set_param(name.encode(), int(v)) == 0, L.last_error()

    def heap_used(self):
        used = ctypes.c_size_t()
        assert self.lib.b200mpi_heap_info(None, ctypes.byref(used), None) == 0, L.last_error()
        return used.value

    def launches(self):
        return self.lib.b200mpi_launch_count()

    def buf(self, storage, dt, count, call, body=None):
        """A guarded buffer of `count` elements in `storage` (a _p2p_plan.STORAGES name)."""
        base, mis = storage.split("+")[0], storage.endswith("+mis")
        off = MISALIGN[DT[dt].itemsize] if mis else 0
        return Buf(base, DT[dt], count, off, self.rank, call, body=body)

    def message(self, dt, count, call):
        return F.gen_values(DT[dt], 1, count, call)[0]


def ptr(b, count):
    """The pointer a caller passes for `count` elements of b: NULL for an empty message."""
    return b.ptr() if count else None


def fail(what, rc):
    raise AssertionError("%s: rc=%d %s" % (what, rc, L.last_error()))


def post(R, b, count, dt, dest, tag, isend):
    fn = R.lib.b200mpi_isend if isend else R.lib.b200mpi_send
    return fn(ptr(b, count), count, CODE[dt], dest, tag, b.memkind)


def recv(R, b, cap, dt, src, tag):
    got = ctypes.c_size_t(12345)
    rc = R.lib.b200mpi_recv(b.ptr() if cap else None, cap, ctypes.byref(got), CODE[dt], src, tag, b.memkind)
    return rc, got.value


def send_side(R, case, dest, tag, call, what, check_launches=True):
    """Send (or Isend and Wait) one planned message; checks the heap, the launches and the buffer."""
    x = R.message(case.dtype, case.count, call)
    b = R.buf(case.send, case.dtype, case.count, call, body=x)
    used, l0 = R.heap_used(), R.launches()
    rc = post(R, b, case.count, case.dtype, dest, tag, case.isend)
    if rc:
        fail(what + " [send]", rc)
    if case.isend and (rc := R.lib.b200mpi_wait(dest, tag)):
        fail(what + " [wait]", rc)
    sp, _ = case.plans()
    assert R.heap_used() == used, "%s: the sender's heap holds %d bytes more after the call" % (what, R.heap_used() - used)
    if check_launches:
        assert R.launches() - l0 == sp.launches, "%s: the sender launched %d kernels, its layout %s launches %d" % (what, R.launches() - l0, sp, sp.launches)
    F.check(b, what + " [send must be unchanged]")
    b.free()


def recv_side(R, case, src, tag, call, what, check_launches=True):
    """Receive one planned message into a buffer with room for 3 more elements; checks the heap, the
    launches, the count and every byte of the buffer."""
    x = R.message(case.dtype, case.count, call)
    b = R.buf(case.recv, case.dtype, case.count + 3, call + 1)
    used, l0 = R.heap_used(), R.launches()
    rc, got = recv(R, b, case.count + 3, case.dtype, src, tag)
    if rc:
        fail(what + " [recv]", rc)
    _, rp = case.plans()
    assert got == case.count, "%s: received %d elements" % (what, got)
    assert R.heap_used() == used, "%s: the receiver's heap holds %d bytes more after the call" % (what, R.heap_used() - used)
    if check_launches:
        assert R.launches() - l0 == rp.launches, "%s: the receiver launched %d kernels, its layout %s launches %d" % (what, R.launches() - l0, rp, rp.launches)
    b.set_body(x)
    F.check(b, what + " [recv: the message, then 3 elements that must not be written]")
    b.free()


def run_case(R, src, dst, case, tag, part):
    """Both sides of one planned case on the ranks it names, each under its own p2p_fast and stage_chunk."""
    call = R.next_call(part)
    pair = case.pair()
    what = "%s %d->%d %s pair=%s" % (part, src, dst, case, pair)
    if R.rank == src:
        R.set("p2p_fast", case.send_fast)
        R.set("stage_chunk", case.stage_chunk)
        send_side(R, case, dst, tag, call, what)
    if R.rank == dst:
        R.set("p2p_fast", case.recv_fast)
        R.set("stage_chunk", case.recv_stage_chunk or case.stage_chunk)
        recv_side(R, case, src, tag, call, what)
    if R.rank in (src, dst):
        key = "%s|%s" % pair
        R.pairs[key] = R.pairs.get(key, 0) + 1


# ---- parts --------------------------------------------------------------------------------------
def part_matrix(R):
    """Every sender storage against every receiver storage, Send and Isend, p2p_fast {on, off} per side,
    the planner's boundary counts over u8, f32, f64 and i64; in a world of 3, every third case from rank
    0 to rank 2 (not its neighbour)."""
    cases = P.matrix() if R.n == 2 else P.matrix(R.n, 0, 2, stride=3)
    for i, (src, dst, case) in enumerate(cases):
        run_case(R, src, dst, case, 10 + i % 7, "matrix")


def part_big(R):
    """big_cases, between ranks 0 and 1."""
    for i, case in enumerate(P.big_cases()):
        run_case(R, 0, 1, case, 30 + i, "big")


# Sender layouts of the error and self-send parts: (layout, Case) at stage_chunk 256 KiB.  The rings
# hold 9 chunks, so that a sender that filled all 4 regions blocks on `done`.
LAYOUT_CASES = (
    ("direct", P.Case("heap+mis", "pinned", False, False, True, "f32", 300001)),
    ("whole/bounce", P.Case("pageable", "torch", False, True, True, "f64", 100001)),
    ("whole/memcpy", P.Case("pinned", "pageable", True, False, False, "i64", 600001)),
    ("whole/kernel", P.Case("torch+mis", "heap", True, True, True, "u8", 3 * P.MB + 5)),
    ("ring/memcpy", P.Case("pageable", "torch+mis", False, False, False, "f32", (2 * P.MB + 4) // 4)),
    ("ring/kernel", P.Case("torch", "pageable", False, False, True, "u8", 2 * P.MB + 1)),
)


def part_errors(R):
    """Truncation and a dtype mismatch against every sender layout, rank 0 sending to rank 1; the ring
    senders have filled all their regions and wait on `done` when the receiver refuses the message.
    Truncation: B200MPI_ERR_TRUNCATE, count_out is the message's count, nothing written, no heap held;
    the retry receives every byte.  Mismatch: B200MPI_ERR_ARG, nothing written, the Send (or Wait)
    returns 0, both heaps at their baseline, and the next message on the tag arrives intact."""
    R.set("stage_chunk", 256 * P.KB)
    for li, (layout, case) in enumerate(LAYOUT_CASES):
        assert case.pair()[0] == layout, (layout, case.pair())
        tag = 50 + li
        for err in ("truncate", "mismatch"):
            call = R.next_call("errors")
            what = "%s against a %s sender %s" % (err, layout, case)
            R.set("p2p_fast", case.send_fast if R.rank == 0 else case.recv_fast)
            if R.rank == 0:
                send_side(R, case, 1, tag, call, what, check_launches=err == "truncate")
                if err == "mismatch":
                    send_side(R, case, 1, tag, call + 1000, what + " [the next message]")
            elif R.rank == 1:
                time.sleep(0.5)  # the ring senders fill their 4 regions meanwhile
                if err == "truncate":
                    dt, cap, want = case.dtype, case.count - 1, L.ERR_TRUNCATE
                else:
                    dt = "i64" if case.dtype != "i64" else "f64"
                    cap, want = case.count * case.es // DT[dt].itemsize + 3, L.ERR_ARG
                small = R.buf(case.recv, dt, cap, call + 7)
                used, l0 = R.heap_used(), R.launches()
                rc, got = recv(R, small, cap, dt, 0, tag)
                assert rc == want and got == case.count, "%s: rc=%d count_out=%d (%s)" % (what, rc, got, L.last_error())
                assert R.heap_used() == used and R.launches() == l0, "%s: the refused receive held heap or launched" % what
                F.check(small, what + " [the refused receive must write nothing]")
                small.free()
                recv_side(R, case, 0, tag, call if err == "truncate" else call + 1000, what + " [retry]" if err == "truncate" else what + " [the next message]")
            mpi.Barrier()


def part_self(R):
    """Self-sends in every sender layout on every rank: a Send from a thread with Receive on the main
    thread, and Isend, Receive and Wait on one thread.  Both sides' launches add up in this process."""
    R.set("stage_chunk", 256 * P.KB)
    me = R.rank
    for li, (layout, case) in enumerate(LAYOUT_CASES):
        for fast in (True, False):
            c = P.Case(case.send, case.recv, case.isend, fast, fast, case.dtype, case.count)
            R.set("p2p_fast", fast)
            call = R.next_call("self")
            what = "self-send %s on rank %d" % (c, me)
            sp, rp = c.plans()
            x = R.message(c.dtype, c.count, call)
            s = R.buf(c.send, c.dtype, c.count, call, body=x)
            r = R.buf(c.recv, c.dtype, c.count + 3, call + 1)
            used, l0 = R.heap_used(), R.launches()
            tag = 70 + li
            if c.isend:
                rc = post(R, s, c.count, c.dtype, me, tag, True)
                if rc:
                    fail(what + " [isend]", rc)
                rc, got = recv(R, r, c.count + 3, c.dtype, me, tag)
                if rc:
                    fail(what + " [recv]", rc)
                if (rc := R.lib.b200mpi_wait(me, tag)):
                    fail(what + " [wait]", rc)
            else:
                out = {}
                t = threading.Thread(target=lambda: out.setdefault("rc", post(R, s, c.count, c.dtype, me, tag, False)))
                t.start()
                rc, got = recv(R, r, c.count + 3, c.dtype, me, tag)
                t.join()
                if out["rc"]:
                    fail(what + " [send]", out["rc"])
                if rc:
                    fail(what + " [recv]", rc)
            assert got == c.count, (what, got)
            assert R.heap_used() == used, "%s: the heap holds %d bytes more" % (what, R.heap_used() - used)
            assert R.launches() - l0 == sp.launches + rp.launches, "%s: %d launches, planned %s + %s" % (what, R.launches() - l0, sp, rp)
            F.check(s, what + " [send must be unchanged]")
            r.set_body(x)
            F.check(r, what + " [recv]")
            s.free()
            r.free()
            key = "%s|%s" % c.pair()
            R.pairs[key] = R.pairs.get(key, 0) + 1


def part_depth(R):
    """16 outstanding Isends from rank 0 to rank 1, received in reverse tag order; with every message
    received but none waited for, a 17th Isend finds no free mailbox slot within a 500 ms watchdog.
    The Waits, in shuffled order, succeed; then nothing is held and the 17th tag works."""
    tags = list(range(100, 100 + P.SLOTS_PER_PAIR))
    extra = 100 + P.SLOTS_PER_PAIR
    cases = [P.Case(("pageable", "pinned", "torch", "heap")[t % 4], "pageable", True, True, True, "f32", 1000 * t + 1) for t in tags]
    R.set("p2p_fast", 1)
    base = R.call
    if R.rank == 0:
        used = R.heap_used()
        bufs = []
        for t, c in zip(tags, cases):
            b = R.buf(c.send, c.dtype, c.count, base + t, body=R.message(c.dtype, c.count, base + t))
            if (rc := post(R, b, c.count, c.dtype, 1, t, True)):
                fail("isend tag %d of %d" % (t, len(tags)), rc)
            bufs.append(b)
        mpi.Barrier()  # rank 1 has received all 16
        wd = L.get_param("watchdog_ms")
        R.set("watchdog_ms", 500)
        x = np.zeros(10, dtype=np.float32)
        t0 = time.time()
        rc = R.lib.b200mpi_isend(x.ctypes.data, 10, L.F32, 1, extra, L.HOST)
        R.set("watchdog_ms", wd)
        assert rc == L.ERR_TIMEOUT and "no free mailbox slot" in L.last_error(), (rc, L.last_error())
        assert time.time() - t0 < 30
        order = list(range(len(tags)))
        random.Random(7).shuffle(order)
        for k in order:
            if (rc := R.lib.b200mpi_wait(1, tags[k])):
                fail("wait tag %d" % tags[k], rc)
        for b in bufs:
            F.check(b, "isend depth [send must be unchanged]")
            b.free()
        assert R.heap_used() == used, "isend depth: %d bytes of staging left behind" % (R.heap_used() - used)
        c = P.Case("pageable", "pageable", True, True, True, "f32", 4097)
        send_side(R, c, 1, extra, base + extra, "the 17th tag after the Waits")
    elif R.rank == 1:
        for t, c in reversed(list(zip(tags, cases))):
            recv_side(R, c, 0, t, base + t, "isend depth, tag %d" % t, check_launches=False)
        mpi.Barrier()
        recv_side(R, P.Case("pageable", "pageable", True, True, True, "f32", 4097), 0, extra, base + extra, "the 17th tag after the Waits")
    R.call = base + extra + 1
    R.done["depth"] = len(tags) + 1


# ---- heap pressure ------------------------------------------------------------------------------
def largest_block(R):
    """The largest block Heap::alloc can give now (found by trying)."""
    total = ctypes.c_size_t()
    R.lib.b200mpi_heap_info(ctypes.byref(total), None, None)
    lo, hi, p = 0, total.value, ctypes.c_void_p()
    while hi - lo > P.HEAP_ALIGN:
        mid = (lo + hi) // 2
        if R.lib.b200mpi_alloc(mid, ctypes.byref(p)) == 0:
            R.lib.b200mpi_free(p)
            lo = mid
        else:
            hi = mid
    return lo


def fill_heap(R, leave):
    """Allocate this rank's heap until the largest free block is `leave` bytes (0: under 4 KiB)."""
    blocks, p = [], ctypes.c_void_p()
    hole = None
    if leave:
        assert R.lib.b200mpi_alloc(leave, ctypes.byref(p)) == 0, L.last_error()
        hole = p.value
    while (size := largest_block(R)) >= 4096:
        assert R.lib.b200mpi_alloc(size, ctypes.byref(p)) == 0, L.last_error()
        blocks.append(p.value)
    if hole:
        R.lib.b200mpi_free(hole)
    return blocks


def free_blocks(R, blocks):
    for b in blocks:
        assert R.lib.b200mpi_free(b) == 0, L.last_error()


# Heap pressure: a world of 2 with a 256 MiB heap, rank 1 at stage_chunk 1 MiB, p2p_fast off.
PRESSURE = {
    "a1": P.Case("heap", "pageable", False, False, False, "u8", 96 * P.MB + 5, P.STAGE_CHUNK, P.MB),
    "a2": P.Case("pageable", "pinned", True, False, False, "u8", 96 * P.MB + 5, P.STAGE_CHUNK, P.MB),
    "b": P.Case("heap", "pageable", False, False, False, "f32", 2 * P.MB + 1, P.STAGE_CHUNK, P.MB),
    "c": P.Case("pageable", "torch", True, False, False, "u8", 16 * P.MB + 1, P.STAGE_CHUNK, P.MB),
}


def pressure_setup(R):
    R.set("p2p_fast", 0)
    R.set("stage_chunk", P.MB if R.rank == 1 else P.STAGE_CHUNK)
    return R.next_call("pressure")


def part_pressure_a(R):
    """96 MiB from a heap buffer (a direct post, one chunk) and from a pageable Isend (one staged chunk)
    reach a pageable and a pinned receiver that has 8 MiB of heap free: it pulls 1 MiB units."""
    call = pressure_setup(R)
    a1, a2 = PRESSURE["a1"], PRESSURE["a2"]
    if R.rank == 0:
        send_side(R, a1, 1, 1, call, "pressure (a) heap send")
        send_side(R, a2, 1, 2, call + 1, "pressure (a) pageable isend")
    elif R.rank == 1:
        used = R.heap_used()
        blocks = fill_heap(R, 8 * P.MB)
        recv_side(R, a1, 0, 1, call, "pressure (a) heap send into pageable, 8 MiB of heap free")
        recv_side(R, a2, 0, 2, call + 1, "pressure (a) pageable isend into pinned, 8 MiB of heap free")
        free_blocks(R, blocks)
        assert R.heap_used() == used


def part_pressure_b(R):
    """A host receive with less than one stage_chunk of heap free fails with B200MPI_ERR_NOMEM, count_out
    set and nothing written.  The message stays posted: once the heap is freed it arrives intact (the
    retry has a 3 s watchdog, so a message that was lost fails it at once), and the Send returns then."""
    call = pressure_setup(R)
    b = PRESSURE["b"]
    if R.rank == 0:
        send_side(R, b, 1, 3, call, "pressure (b) heap send")
    elif R.rank == 1:
        used = R.heap_used()
        blocks = fill_heap(R, 0)
        r = R.buf(b.recv, b.dtype, b.count + 3, call + 7)
        rc, got = recv(R, r, b.count + 3, b.dtype, 0, 3)
        assert rc == L.ERR_NOMEM and got == b.count, "pressure (b): rc=%d count_out=%d (%s)" % (rc, got, L.last_error())
        F.check(r, "pressure (b) [a receive that failed for heap must write nothing]")
        r.free()
        free_blocks(R, blocks)
        assert R.heap_used() == used
        wd = L.get_param("watchdog_ms")
        R.set("watchdog_ms", 3000)
        try:
            recv_side(R, b, 0, 3, call, "pressure (b) the retry after freeing the heap")
        finally:
            R.set("watchdog_ms", wd)


def part_pressure_c(R):
    """An Isend larger than the sender's free heap fails with B200MPI_ERR_NOMEM; its slot and tag are
    released, nothing is pending, and the next Isend on the tag works."""
    call = pressure_setup(R)
    c = PRESSURE["c"]
    if R.rank == 0:
        used = R.heap_used()
        blocks = fill_heap(R, 8 * P.MB)
        s = R.buf(c.send, c.dtype, c.count, call, body=R.message(c.dtype, c.count, call))
        rc = post(R, s, c.count, c.dtype, 1, 4, True)
        assert rc == L.ERR_NOMEM, "pressure (c): an Isend larger than the free heap gave rc=%d (%s)" % (rc, L.last_error())
        free_blocks(R, blocks)
        assert R.heap_used() == used, "pressure (c): the failed Isend held %d bytes" % (R.heap_used() - used)
        assert R.lib.b200mpi_wait(1, 4) == L.ERR_ARG, "pressure (c): the failed Isend left a pending send"
        F.check(s, "pressure (c) [send must be unchanged]")
        s.free()
        send_side(R, c, 1, 4, call, "pressure (c) the Isend again")
    elif R.rank == 1:
        recv_side(R, c, 0, 4, call, "pressure (c)")


# ---- concurrency --------------------------------------------------------------------------------
# (send storage, recv storage, isend, dtype, count): host sends of at most 4 MiB first
HOST_SPECS = (("pageable", "pinned", False, "f32", 200001), ("pinned", "pageable", True, "u8", P.MB + 3),
              ("torchpin", "torch+mis", False, "f64", 70001), ("pageable", "heap+mis", True, "i64", 300001),
              ("pinned", "torchpin", False, "u8", 4 * P.MB - 1))
DEVICE_SPECS = (("torch+mis", "pageable", False, "f64", 90001), ("heap", "torchpin", False, "i64", 150001),
                ("heap+mis", "torch", True, "f32", 50001), ("torch", "heap", False, "u8", 2 * P.MB + 3))


def conc_spec(n, src, dst, t, tags):
    """The message src sends dst with tag index t: tag indexes 0 and 1 are host slices, the rest device
    buffers, the specs rotating per (pair, tag); in a world of 8, at most 1 MiB."""
    specs = HOST_SPECS if t < 2 else DEVICE_SPECS
    s, r, isend, dt, count = specs[(src + 2 * dst + 3 * t) % len(specs)]
    if n >= 8:
        count = min(count, P.MB // DT[dt].itemsize + 1)
    return P.Case(s, r, isend, True, True, dt, count)


def part_concurrent(R, tags):
    """Every ordered pair of ranks, self included, exchanges `tags` messages at once from threads, with
    p2p_fast on: each rank has 2n host-slice sends of at most 4 MiB in flight, more than the 4 mapped
    bounces, so some of them fall back to the ring.  Every buffer is checked; the heap is at its
    baseline at the end."""
    n, me = R.n, R.rank
    R.set("p2p_fast", 1)
    R.set("stage_chunk", 256 * P.KB)
    used = R.heap_used()
    base = R.call
    jobs, sends, recvs, errors = [], [], [], []

    def cid(src, dst, t):
        return base + 1 + 2 * ((src * n + dst) * tags + t)

    for d in range(n):
        for t in range(tags):
            c = conc_spec(n, me, d, t, tags)
            sends.append((d, t, c, R.buf(c.send, c.dtype, c.count, cid(me, d, t), body=R.message(c.dtype, c.count, cid(me, d, t)))))
    for s in range(n):
        for t in range(tags):
            c = conc_spec(n, s, me, t, tags)
            recvs.append((s, t, c, R.buf(c.recv, c.dtype, c.count + 3, cid(s, me, t) + 1)))

    def do_send(d, t, c, b):
        try:
            if (rc := post(R, b, c.count, c.dtype, d, 200 + t, c.isend)):
                fail("send %d->%d tag %d %s" % (me, d, t, c), rc)
            if c.isend and (rc := R.lib.b200mpi_wait(d, 200 + t)):
                fail("wait %d->%d tag %d %s" % (me, d, t, c), rc)
        except Exception as e:  # noqa: BLE001
            errors.append(str(e))

    def do_recv(s, t, c, b):
        try:
            rc, got = recv(R, b, c.count + 3, c.dtype, s, 200 + t)
            if rc:
                fail("recv %d->%d tag %d %s" % (s, me, t, c), rc)
            assert got == c.count
        except Exception as e:  # noqa: BLE001
            errors.append(str(e))

    mpi.Barrier()
    for x in sends:
        jobs.append(threading.Thread(target=do_send, args=x))
    for x in recvs:
        jobs.append(threading.Thread(target=do_recv, args=x))
    random.Random(me).shuffle(jobs)
    for j in jobs:
        j.start()
    for j in jobs:
        j.join()
    if errors:
        raise AssertionError("%d concurrent calls failed, first: %s" % (len(errors), errors[0]))
    for d, t, c, b in sends:
        F.check(b, "concurrent send %d->%d tag %d %s [send must be unchanged]" % (me, d, t, c))
        b.free()
    for s, t, c, b in recvs:
        b.set_body(R.message(c.dtype, c.count, cid(s, me, t)))
        F.check(b, "concurrent recv %d->%d tag %d %s" % (s, me, t, c))
        b.free()
    assert R.heap_used() == used, "concurrent: %d bytes of heap held after every call returned" % (R.heap_used() - used)
    host = sum(1 for _, _, c, _ in sends if P.STORAGES[c.send][0] == "host" and c.nbytes <= P.BOUNCE_BYTES)
    R.call = cid(n - 1, n - 1, tags - 1) + 2
    R.done["concurrent"] = len(sends) + len(recvs)
    return host


PARTS = ("matrix", "big", "errors", "self", "depth", "pressure_a", "pressure_b", "pressure_c", "concurrent")


def scenario_p2p(a, opts):
    R = Run()
    secs, out = {}, {}
    for name in opts.parts.split(","):
        assert name in PARTS, name
        t0 = time.time()
        if name == "concurrent":
            out["host_sends_in_flight"] = part_concurrent(R, opts.tags)
        else:
            globals()["part_" + name](R)
        mpi.Barrier()
        secs[name] = round(time.time() - t0, 2)
    out.update({"checked": R.call, "by_part": R.done, "seconds": secs, "pairs": R.pairs})
    return out


def parse_options(argv):
    ap = argparse.ArgumentParser(add_help=False)
    ap.add_argument("--parts", default="matrix")
    ap.add_argument("--tags", type=int, default=3, help="messages per ordered pair in part concurrent")
    return ap.parse_known_args(argv)


if __name__ == "__main__":
    opts, rest = parse_options(sys.argv[1:])
    sys.argv = [sys.argv[0]] + rest
    W.SCENARIOS["p2p"] = lambda a: scenario_p2p(a, opts)
    W.main()
