"""One rank of a test world for the passive-target calls (Lock, Unlock, GetAccumulate, FetchAndOp,
CompareAndSwap).  Usage as _worker.py: _rma_atomic_worker.py <scenario> --out FILE [scenario args]
-mpi-* flags.  Windows, origins and results are guarded views (_kinds_worker.Buf); fetched values and
windows are compared with the model (_rma_atomic_ref) byte for byte, and every window allocation,
guards included, is checked after a Barrier that follows the last call into it (every call has
completed when it returns)."""
import ctypes
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _footprint_worker as F  # noqa: E402
import _kinds_worker as K  # noqa: E402
import _rma_atomic_ref as A  # noqa: E402
import _worker as W  # noqa: E402
from _worker import L, mpi  # noqa: E402

DTS = (np.float32, np.float64, np.int64)


class Wnd:
    """A guarded window of `count` elements of dt at byte `off` past the guard on every rank, created
    collectively with body `init(rank)`.  `images[r]` is the model of rank r's window body (bytes)."""

    def __init__(self, dt, count, off, key, init):
        self.dt, self.count = np.dtype(dt), count
        self.rank, self.n = mpi.Rank(), mpi.Size()
        self.images = [np.ascontiguousarray(init(r), dtype=dt).view(np.uint8).copy() for r in range(self.n)]
        self.buf = K.Buf("heap", dt, count, off, self.rank, key, body=init(self.rank))
        self.win = mpi.WinCreate(self.buf.view)

    def model(self, r):
        return self.images[r].view(self.dt)

    def check(self, what, nan_equal=False):
        """After a Barrier that follows every call into the window: this rank's window is its image,
        the guards their pattern."""
        got = self.buf.read()
        body = got[self.buf.head:self.buf.head + self.buf.nbody].view(self.dt)
        assert A.same_bits(body, self.model(self.rank), nan_equal), (what, body[:8], self.model(self.rank)[:8])
        self.buf.set_body(body)
        F.check(self.buf, what + " [guards of rank %d's window]" % self.rank)

    def free(self):
        self.win.Free()
        self.buf.free()


def allgather_i64(vals):
    send = np.ascontiguousarray(vals, dtype=np.int64)
    recv = np.empty(send.size * mpi.Size(), dtype=np.int64)
    mpi.Allgather(send, recv)
    return recv.reshape(mpi.Size(), send.size)


def scenario_ra_tickets(a):
    """Every rank takes K tickets with FetchAndOp(SUM, 1) on rank 0's counter, then K on a counter of
    every rank; the fetched values over all ranks are exactly 0 .. nK-1 and every counter ends at nK.
    Then the same with f64 on small integers (exact)."""
    rank, n = mpi.Rank(), mpi.Size()
    K_ = 40
    done = 0
    for dt, one in ((np.int64, np.int64(1)), (np.float64, np.float64(1.0))):
        w = Wnd(dt, n + 1, 8, 11 + done, lambda r: np.zeros(n + 1, dtype=dt))
        got = [w.win.FetchAndOp(one, 0, 0) for _ in range(K_)]
        for t in range(n):
            got += [w.win.FetchAndOp(one, t, 1 + t) for _ in range(K_)]
        assert all(type(g) is type(one) for g in got), [type(g) for g in got[:3]]
        allv = allgather_i64([int(g) for g in got])
        for c in range(n + 1):
            seen = sorted(allv[:, c * K_:(c + 1) * K_].ravel().tolist())
            assert seen == list(range(n * K_)), ("tickets", np.dtype(dt), c, seen[:10])
        mpi.Barrier()
        for c in range(n + 1):
            final = w.win.FetchAndOp(one, 0 if c == 0 else c - 1, c, op=A.NO_OP)
            assert final == n * K_, ("final counter", c, final)
        body = np.zeros(n + 1, dtype=dt)
        body[0] = n * K_ if rank == 0 else 0
        body[1 + rank] = n * K_
        w.images[rank] = body.view(np.uint8).copy()
        mpi.Barrier()
        w.check("tickets %s" % np.dtype(dt))
        w.free()
        done += 1
    mpi.Barrier()
    return {"checked": done}


def scenario_ra_election(a):
    """Every rank calls CompareAndSwap(rank, compare=-1) on C cells of every rank's window: per cell,
    exactly one rank fetched -1, every other rank fetched that winner, and the cell holds it."""
    rank, n = mpi.Rank(), mpi.Size()
    C = 5
    w = Wnd(np.int64, C, 16, 21, lambda r: np.full(C, -1, dtype=np.int64))
    got = []
    for i in range(n):
        t = (rank + i) % n
        for c in range(C):
            got.append((t, c, int(w.win.CompareAndSwap(rank, -1, t, c))))
    order = sorted(got)
    allv = allgather_i64([g[2] for g in order])  # [rank][t * C + c]
    mpi.Barrier()
    winners = np.empty((n, C), dtype=np.int64)
    for t in range(n):
        for c in range(C):
            col = allv[:, t * C + c]
            won = [r for r in range(n) if col[r] == -1]
            assert len(won) == 1, ("election", t, c, col.tolist())
            winners[t, c] = won[0]
            assert all(col[r] == won[0] for r in range(n) if r != won[0]), ("losers fetch the winner", t, c, col.tolist())
            assert w.win.FetchAndOp(0, t, c, op=A.NO_OP) == won[0], ("cell holds the winner", t, c)
    w.images[rank] = winners[rank].view(np.uint8).copy()
    mpi.Barrier()
    w.check("election")
    w.free()
    mpi.Barrier()
    return {"checked": n * C}


def scenario_ra_swap(a):
    """Every rank swaps its own values into the same elements of rank 0's window with REPLACE, through
    GetAccumulate (host and heap results) and FetchAndOp; per element, all fetched values plus the final
    value are a permutation of the initial value and all contributions."""
    rank, n = mpi.Rank(), mpi.Size()
    E, S = 6, 12
    done = 0
    for dt in (np.int64, np.float32):
        w = Wnd(dt, E, 4 if dt == np.float32 else 8, 31 + done, lambda r: (np.arange(E) * -1 - 1).astype(dt))
        mine = lambda s: (1000 * (rank + 1) + 10 * s + np.arange(E)).astype(dt)  # noqa: E731
        fetched = []
        for s in range(S):
            if s % 3 == 2:
                fetched.append([w.win.FetchAndOp(mine(s)[e], 0, e, op=A.REPLACE) for e in range(E)])
                continue
            storage = "heap" if s % 3 == 0 else "pageable"
            o = K.Buf(storage, dt, E, 4 * (s % 2), rank, 300 + s, body=mine(s))
            res = K.Buf(storage, dt, E, 8, rank, 400 + s)
            w.win.GetAccumulate(o.view, res.view, 0, 0, op=A.REPLACE)
            got = res.read()[res.head:res.head + res.nbody].view(dt).copy()
            F.check(o, "swap origin unchanged")
            res.set_body(got)
            F.check(res, "swap result guards")
            fetched.append(got.tolist())
            o.free()
            res.free()
        allv = allgather_i64(np.array(fetched, dtype=dt).astype(np.int64).ravel())
        mpi.Barrier()
        final = [w.win.FetchAndOp(dt(0), 0, e, op=A.NO_OP) for e in range(E)]
        for e in range(E):
            got = sorted(allv.reshape(n, S, E)[:, :, e].ravel().tolist() + [int(final[e])])
            want = sorted([-(e + 1)] + [int(1000 * (r + 1) + 10 * s + e) for r in range(n) for s in range(S)])
            assert got == want, ("swap chain", np.dtype(dt), e)
        if rank == 0:
            w.images[0] = np.array(final, dtype=dt).view(np.uint8).copy()
        mpi.Barrier()
        w.check("swap %s" % np.dtype(dt))
        w.free()
        done += 1
    mpi.Barrier()
    return {"checked": done}


def special_values(dt, salt):
    """16 values: NaN, zeros of both signs, subnormals, infinities and ordinary numbers (floats), or
    int64 extremes; rotated by salt."""
    if np.dtype(dt) == np.int64:
        i = np.iinfo(np.int64)
        v = np.array([i.max, i.min, -1, 0, 1, i.max - 3, i.min + 2, 7, -7, 1 << 40, -(1 << 40), 12345, 99, -100, 5, i.max], dtype=np.int64)
    else:
        fi = np.finfo(dt)
        sub = fi.tiny / 4
        v = np.array([np.nan, 0.0, -0.0, sub, -sub, fi.tiny, 1.5 * fi.tiny, -fi.tiny, np.inf, -np.inf, 1.0, -2.5, 3.0, 1e-3, 7.25, np.nan],
                     dtype=dt)
    return np.roll(v, salt)


def scenario_ra_rules(a):
    """One rank at a time, against the model byte for byte: every dtype and op of GetAccumulate on
    special values (NaN, subnormals, zeros, infinities, int64 extremes), with origins and results on the
    heap, on the heap off element alignment, in pinned and pageable host memory, in torch memory, and in
    place; FetchAndOp of every dtype and op; Accumulate with REPLACE.  A SUM into a NaN compares NaN
    as NaN (its payload is the hardware's); every fetched value is the previous bits exactly."""
    rank, n = mpi.Rank(), mpi.Size()
    N = 16
    layouts = ("heap", "heap_mis", "pinned", "pageable", "torch", "inplace_heap", "inplace_host")
    done = 0
    for j, dt in enumerate(DTS):
        es = np.dtype(dt).itemsize
        w = Wnd(dt, N + 3, (es * j) % 16, 51 + j, lambda r: np.zeros(N + 3, dtype=dt))
        for turn in range(n):
            if rank == turn:
                t = (rank + 1) % n
                for k, (opname, op) in enumerate(A.OPS.items()):
                    lay = layouts[(k + j + turn) % len(layouts)]
                    init, orig = special_values(dt, k), special_values(dt, 5 + 3 * k)
                    disp = 1 + k % 3
                    w.win.Put(init, t, disp)
                    want_fetch, want_new = A.fetch_op(init, orig, op)
                    storage = {"heap_mis": "heap", "inplace_heap": "heap", "inplace_host": "pageable"}.get(lay, lay)
                    off = (1 + k) % es + 1 if lay == "heap_mis" else 4 * (k % 4)
                    o = K.Buf(storage, dt, N, off, rank, 600 + k, body=orig)
                    if lay.startswith("inplace"):
                        w.win.GetAccumulate(o.view, o.view, t, disp, op=op)
                        got = o.read()[o.head:o.head + o.nbody].view(dt).copy()
                        assert A.same_bits(got, want_fetch), ("in place fetch", np.dtype(dt), opname, lay, got, want_fetch)
                        o.set_body(got)
                        F.check(o, "in place guards")
                    else:
                        res = K.Buf(storage, dt, N, (off + es) % 16 if lay != "heap_mis" else off + 2, rank, 700 + k)
                        w.win.GetAccumulate(None if op == A.NO_OP and k % 2 else o.view, res.view, t, disp, op=op)
                        got = res.read()[res.head:res.head + res.nbody].view(dt).copy()
                        assert A.same_bits(got, want_fetch), ("fetch", np.dtype(dt), opname, lay, got, want_fetch)
                        res.set_body(got)
                        F.check(res, "result guards")
                        F.check(o, "origin unchanged")
                        res.free()
                    o.free()
                    now = w.win.Get(np.empty(N, dtype=dt), t, disp)
                    assert A.same_bits(now, want_new, nan_equal=op == A.SUM), ("target", np.dtype(dt), opname, lay, now, want_new)
                    # FetchAndOp of one element, the same rules
                    for e in range(0, N, 5):
                        w.win.Put(init[e:e + 1], t, disp)
                        old = w.win.FetchAndOp(orig[e], t, disp, op=op)
                        assert A.same_bits(np.array([old], dtype=dt), init[e:e + 1]), ("fetch_and_op", np.dtype(dt), opname, e, old, init[e])
                        now1 = w.win.Get(np.empty(1, dtype=dt), t, disp)
                        assert A.same_bits(now1, A.apply(init[e:e + 1], orig[e:e + 1], op), nan_equal=op == A.SUM), ("fetch_and_op target", opname, e)
                    done += 1
                # Accumulate with REPLACE, from a heap origin off its alignment
                vals = special_values(dt, 9)
                o = K.Buf("heap", dt, N, 3, rank, 800, body=vals)
                w.win.Accumulate(o.view, t, 2, op=A.REPLACE)
                o.free()
                now = w.win.Get(np.empty(N, dtype=dt), t, 2)
                assert A.same_bits(now, vals), ("accumulate replace", np.dtype(dt))
                body = np.zeros(N + 3, dtype=dt)
                body[2:2 + N] = vals
                w.win.Put(body, t, 0)
                w.images[t] = body.view(np.uint8).copy()
                done += 1
            else:
                t = (turn + 1) % n
                body = np.zeros(N + 3, dtype=dt)
                body[2:2 + N] = special_values(dt, 9)
                w.images[t] = body.view(np.uint8).copy()
            mpi.Barrier()
        w.check("rules %s" % np.dtype(dt))
        w.free()
    mpi.Barrier()
    return {"checked": done}


def scenario_ra_mutex(a):
    """R rounds: each rank visits every target in a rotating order (itself included) and, under an
    exclusive lock, Gets the target's record, checks that its elements agree, adds 1 to each and Puts it
    back; between visits it reads another target's record under a shared lock, and every record it sees
    has all its elements equal.  Every record ends at n * R (the model of serial rounds)."""
    rank, n = mpi.Rank(), mpi.Size()
    Rr = 3 if n <= 4 else 2
    Ln = 33
    w = Wnd(np.int64, Ln, 8, 61, lambda r: np.zeros(Ln, dtype=np.int64))
    shared_reads = 0
    for r in range(Rr):
        for j in range(n):
            t = (rank + r + j) % n
            w.win.Lock(t)
            rec = w.win.Get(np.empty(Ln, dtype=np.int64), t, 0)
            assert np.all(rec == rec[0]), ("torn record under an exclusive lock", t, rec)
            w.win.Put(rec + 1, t, 0)
            w.win.Unlock(t)
            s = (rank + r + j + 1) % n
            w.win.Lock(s, mpi.LOCK_SHARED)
            seen = w.win.Get(np.empty(Ln, dtype=np.int64), s, 0)
            w.win.Unlock(s)
            assert np.all(seen == seen[0]), ("torn record under a shared lock", s, seen)
            shared_reads += 1
    mpi.Barrier()
    model = A.locked_rounds(n, Rr, Ln, lambda k, r: [(k + r + j) % n for j in range(n)])
    w.images = [m.view(np.uint8).copy() for m in model]
    w.check("mutex")
    w.free()
    mpi.Barrier()
    return {"checked": n * Rr + shared_reads}


def scenario_ra_counts(a):
    """An uncontended Lock, Unlock, FetchAndOp, CompareAndSwap and a heap GetAccumulate are one launch
    each, take no epoch and leave the heap as it was."""
    lib, rank, n = L.load(), mpi.Rank(), mpi.Size()
    w = Wnd(np.int64, 64, 0, 71, lambda r: np.zeros(64, dtype=np.int64))
    src = mpi.Alloc(16, np.int64).copy_from_host(np.arange(16, dtype=np.int64))
    dst = mpi.Alloc(16, np.int64)
    t = (rank + 1) % n
    mpi.Barrier()
    used = ctypes.c_size_t()
    assert lib.b200mpi_heap_info(None, ctypes.byref(used), None) == 0
    used0, epoch0 = used.value, L.get_param("epoch")
    for name, call in (("lock", lambda: w.win.Lock(t)), ("unlock", lambda: w.win.Unlock(t)),
                       ("fetch_and_op", lambda: w.win.FetchAndOp(5, t, 3)),
                       ("compare_and_swap", lambda: w.win.CompareAndSwap(9, 0, t, 40 + rank)),
                       ("get_accumulate", lambda: w.win.GetAccumulate(src, dst, t, 20))):
        l0 = lib.b200mpi_launch_count()
        call()
        assert lib.b200mpi_launch_count() == l0 + 1, (name, lib.b200mpi_launch_count() - l0)
        assert L.get_param("epoch") == epoch0, (name, "took an epoch")
        assert lib.b200mpi_heap_info(None, ctypes.byref(used), None) == 0 and used.value == used0, (name, "used heap")
    mpi.Barrier()
    dst.free()
    src.free()
    w.free()
    mpi.Barrier()
    return {"checked": 5}


def scenario_ra_errors(a):
    """Every argument error returns its code and writes nothing: locks (twice, without, bad type,
    target out of range, unknown and freed windows), GetAccumulate of u8, CompareAndSwap of f32, NO_OP
    to Accumulate, a result overlapping the origin in part, and Allreduce, Reduce and Scan with ops 3
    and 4.  The window and the buffers are checked afterwards."""
    lib, rank, n = L.load(), mpi.Rank(), mpi.Size()
    w = Wnd(np.float64, 32, 8, 81, lambda r: np.arange(32, dtype=np.float64) + 100 * r)
    gone = mpi.WinCreate(None)
    gone.Free()
    other = mpi.WinCreate(None)  # live, never locked
    wid, t = w.win.id, (rank + 1) % n
    h = np.arange(8, dtype=np.float64)
    h0 = h.copy()
    res = np.full(8, 7.0)
    hp, rp = h.ctypes.data, res.ctypes.data
    i64 = np.array([3], dtype=np.int64)
    f32 = np.array([3], dtype=np.float32)
    ip, fp = i64.ctypes.data, f32.ctypes.data
    x = np.ones(4, dtype=np.float64)
    y = np.zeros(4, dtype=np.float64)
    assert lib.b200mpi_win_lock(L.LOCK_SHARED, t, wid) == 0, L.last_error()
    cases = (
        ("double lock", lambda: lib.b200mpi_win_lock(L.LOCK_EXCLUSIVE, t, wid), L.ERR_ARG),
        ("unlock without a lock", lambda: lib.b200mpi_win_unlock(t, other.id), L.ERR_ARG),
        ("lock type 0", lambda: lib.b200mpi_win_lock(0, rank, wid), L.ERR_ARG),
        ("lock type 3", lambda: lib.b200mpi_win_lock(3, rank, wid), L.ERR_ARG),
        ("lock target = size", lambda: lib.b200mpi_win_lock(L.LOCK_EXCLUSIVE, n, wid), L.ERR_ARG),
        ("lock negative target", lambda: lib.b200mpi_win_lock(L.LOCK_EXCLUSIVE, -1, wid), L.ERR_ARG),
        ("unlock target = size", lambda: lib.b200mpi_win_unlock(n, wid), L.ERR_ARG),
        ("lock unknown window", lambda: lib.b200mpi_win_lock(L.LOCK_EXCLUSIVE, t, wid + 100), L.ERR_ARG),
        ("lock freed window", lambda: lib.b200mpi_win_lock(L.LOCK_EXCLUSIVE, t, gone.id), L.ERR_ARG),
        ("unlock freed window", lambda: lib.b200mpi_win_unlock(t, gone.id), L.ERR_ARG),
        ("u8 get_accumulate", lambda: lib.b200mpi_get_accumulate(hp, rp, 1, L.U8, L.SUM, t, 0, wid, L.HOST), L.ERR_UNSUPPORTED),
        ("u8 fetch_and_op", lambda: lib.b200mpi_fetch_and_op(hp, rp, L.U8, L.SUM, t, 0, wid), L.ERR_UNSUPPORTED),
        ("f32 compare_and_swap", lambda: lib.b200mpi_compare_and_swap(fp, fp, fp, L.F32, t, 0, wid), L.ERR_UNSUPPORTED),
        ("f64 compare_and_swap", lambda: lib.b200mpi_compare_and_swap(hp, hp, rp, L.F64, t, 0, wid), L.ERR_UNSUPPORTED),
        ("u8 compare_and_swap", lambda: lib.b200mpi_compare_and_swap(ip, ip, rp, L.U8, t, 0, wid), L.ERR_UNSUPPORTED),
        ("unknown dtype compare_and_swap", lambda: lib.b200mpi_compare_and_swap(ip, ip, rp, 9, t, 0, wid), L.ERR_ARG),
        ("NO_OP to accumulate", lambda: lib.b200mpi_accumulate(hp, 1, L.F64, L.NO_OP, t, 0, wid, L.HOST), L.ERR_ARG),
        ("op 5 to get_accumulate", lambda: lib.b200mpi_get_accumulate(hp, rp, 1, L.F64, 5, t, 0, wid, L.HOST), L.ERR_ARG),
        ("op -1 to fetch_and_op", lambda: lib.b200mpi_fetch_and_op(hp, rp, L.F64, -1, t, 0, wid), L.ERR_ARG),
        ("partial overlap", lambda: lib.b200mpi_get_accumulate(hp, hp + 8, 4, L.F64, L.SUM, t, 0, wid, L.HOST), L.ERR_ARG),
        ("NULL origin with SUM", lambda: lib.b200mpi_get_accumulate(None, rp, 2, L.F64, L.SUM, t, 0, wid, L.HOST), L.ERR_ARG),
        ("NULL result", lambda: lib.b200mpi_get_accumulate(hp, None, 2, L.F64, L.SUM, t, 0, wid, L.HOST), L.ERR_ARG),
        ("NULL fetch origin", lambda: lib.b200mpi_fetch_and_op(None, rp, L.F64, L.MAX, t, 0, wid), L.ERR_ARG),
        ("NULL cas compare", lambda: lib.b200mpi_compare_and_swap(ip, None, rp, L.I64, t, 0, wid), L.ERR_ARG),
        ("get_accumulate past the window", lambda: lib.b200mpi_get_accumulate(hp, rp, 2, L.F64, L.SUM, t, 31, wid, L.HOST), L.ERR_ARG),
        ("fetch_and_op past the window", lambda: lib.b200mpi_fetch_and_op(hp, rp, L.F64, L.SUM, t, 32, wid), L.ERR_ARG),
        ("get_accumulate target = size", lambda: lib.b200mpi_get_accumulate(hp, rp, 1, L.F64, L.SUM, n, 0, wid, L.HOST), L.ERR_ARG),
        ("get_accumulate bad memkind", lambda: lib.b200mpi_get_accumulate(hp, rp, 1, L.F64, L.SUM, t, 0, wid, 7), L.ERR_ARG),
        ("fetch_and_op unknown window", lambda: lib.b200mpi_fetch_and_op(hp, rp, L.F64, L.SUM, t, 0, gone.id), L.ERR_ARG),
    )
    done = 0
    for name, call, want in cases:
        rc = call()
        assert rc == want, (name, rc, want, L.last_error())
        done += 1
    # the collectives still refuse the one-sided ops
    for op in (L.REPLACE, L.NO_OP):
        for name, call in (("allreduce", lambda: mpi.Allreduce(x, y, op)), ("reduce", lambda: mpi.Reduce(x, y, op, 0)),
                           ("scan", lambda: mpi.Scan(x, y, op))):
            try:
                call()
                raise AssertionError("%s with op %d succeeded" % (name, op))
            except mpi.MpiError as e:
                assert e.code == L.ERR_ARG, (name, op, e.code)
            done += 1
    assert np.all(y == 0), "a refused collective wrote its recv"
    # count 0 is legal and does nothing; NO_OP with a NULL origin fetches
    assert lib.b200mpi_get_accumulate(None, None, 0, L.F64, L.SUM, t, 0, wid, L.HOST) == 0, L.last_error()
    assert lib.b200mpi_get_accumulate(None, rp, 2, L.F64, L.NO_OP, t, 3, wid, L.HOST) == 0, L.last_error()
    assert res[:2].tolist() == [3.0 + 100 * t, 4.0 + 100 * t] and np.all(res[2:] == 7.0), res
    assert np.array_equal(h, h0), "an origin was written"
    assert lib.b200mpi_win_unlock(t, wid) == 0, L.last_error()
    mpi.Barrier()
    w.check("errors: nothing written")
    other.Free()
    w.free()
    mpi.Barrier()
    return {"checked": done + 2}


def scenario_ra_fence_locked(a):
    """Fence and Free by a rank holding a lock: ERR_ARG there, ERR_PEER on every other rank (a world of
    one: ERR_ARG and nothing launched).  The window stays live and the lock held; after the unlock the
    next fence works.  When every rank holds a lock, every rank gets ERR_ARG; then Free works."""
    lib, rank, n = L.load(), mpi.Rank(), mpi.Size()
    w = Wnd(np.int64, 10, 0, 91, lambda r: np.zeros(10, dtype=np.int64))
    holder = n - 1
    if rank == holder:
        w.win.Lock(0)
    for what in ("fence", "free"):
        l0 = lib.b200mpi_launch_count()
        rc = lib.b200mpi_win_fence(w.win.id) if what == "fence" else lib.b200mpi_win_free(w.win.id)
        want = L.ERR_ARG if rank == holder else L.ERR_PEER
        assert rc == want, (what, rc, want, L.last_error())
        if n == 1:
            assert lib.b200mpi_launch_count() == l0, "a world of one launched a fence"
    # still live: atomics and the held lock work
    assert w.win.FetchAndOp(1, 0, 1 + rank) == 0
    if rank == holder:
        w.win.Put(np.array([5], dtype=np.int64), 0, 0)
        w.win.Unlock(0)
    w.win.Fence()
    body = np.zeros(10, dtype=np.int64)
    if rank == 0:
        body[0] = 5
        body[1:1 + n] = 1
    w.images[rank] = body.view(np.uint8).copy()
    w.check("fence against a held lock")
    w.win.Fence()
    # every rank holding a lock: their marks agree, and still every rank is refused
    w.win.Lock(0, mpi.LOCK_SHARED)
    rc = lib.b200mpi_win_fence(w.win.id)
    assert rc == L.ERR_ARG, (rc, L.last_error())
    w.win.Unlock(0)
    w.free()
    mpi.Barrier()
    return {"checked": 5}


def scenario_ra_timeout(a):
    """Rank 0 holds an exclusive lock on its window; rank 1, with watchdog_ms at 2000, gets ERR_TIMEOUT
    from Lock and holds nothing; after rank 0 unlocks, rank 1's Lock succeeds.  Each attempt kernel is
    bounded, so no kernel waits long: this tests the host's deadline."""
    rank = mpi.Rank()
    w = Wnd(np.int64, 4, 0, 93, lambda r: np.zeros(4, dtype=np.int64))
    if rank == 0:
        w.win.Lock(0)
    mpi.Barrier()
    if rank == 1:
        old = L.get_param("watchdog_ms")
        assert L.load().b200mpi_set_param(b"watchdog_ms", 2000) == 0
        t0 = time.time()
        try:
            w.win.Lock(0)
            raise AssertionError("lock granted while rank 0 holds it")
        except mpi.MpiError as e:
            assert e.code == L.ERR_TIMEOUT, (e.code, str(e))
        finally:
            assert L.load().b200mpi_set_param(b"watchdog_ms", old) == 0
        dt = time.time() - t0
        assert 1.9 < dt < 60, dt
        assert L.load().b200mpi_win_unlock(0, w.win.id) == L.ERR_ARG, "the timed-out lock is held"
    mpi.Barrier()
    if rank == 0:
        w.win.Unlock(0)
    mpi.Barrier()
    if rank == 1:
        w.win.Lock(0)
        assert w.win.FetchAndOp(1, 0, 2) == 0
        w.win.Unlock(0)
    mpi.Barrier()
    if rank == 0:
        w.images[0] = np.array([0, 0, 1, 0], dtype=np.int64).view(np.uint8).copy()
    w.check("timeout")
    w.free()
    mpi.Barrier()
    return {"checked": 3}


def scenario_ra_cells(a):
    """One window stays live (and locked by every rank on its neighbour) while a few hundred others are
    created and freed; an exclusive and a shared lock work on every one of them, so the freed windows'
    lock words are handed out again clear."""
    rank, n = mpi.Rank(), mpi.Size()
    keep = Wnd(np.int64, 4, 0, 95, lambda r: np.zeros(4, dtype=np.int64))
    t = (rank + 1) % n
    keep.win.Lock(t, mpi.LOCK_SHARED)
    mem = mpi.Alloc(8, np.int64).copy_from_host(np.zeros(8, dtype=np.int64))
    cycles = 300 if n <= 2 else 120
    for i in range(cycles):
        w = mpi.WinCreate(mem)
        assert w.id > keep.win.id
        w.Lock(t)
        assert w.FetchAndOp(1, t, 0) == i
        w.Unlock(t)
        w.Lock(t, mpi.LOCK_SHARED)
        w.Unlock(t)
        w.Free()
    keep.win.Unlock(t)
    keep.win.Fence()
    assert mem.to_host()[0] == cycles
    mem.free()
    keep.free()
    mpi.Barrier()
    return {"checked": cycles}


def scenario_ra_control_only(a):
    """Control plane only: all five entries refuse with B200MPI_ERR_NO_DEVICE, through the C ABI and the facade."""
    lib = L.load()
    x = np.zeros(4, np.int64)
    p = x.ctypes.data
    assert lib.b200mpi_win_lock(L.LOCK_EXCLUSIVE, 0, 0) == L.ERR_NO_DEVICE
    assert lib.b200mpi_win_unlock(0, 0) == L.ERR_NO_DEVICE
    assert lib.b200mpi_get_accumulate(p, p, 1, L.I64, L.SUM, 0, 0, 0, L.HOST) == L.ERR_NO_DEVICE
    assert lib.b200mpi_fetch_and_op(p, p, L.I64, L.SUM, 0, 0, 0) == L.ERR_NO_DEVICE
    assert lib.b200mpi_compare_and_swap(p, p, p, L.I64, 0, 0, 0) == L.ERR_NO_DEVICE
    w = mpi.Win(0)
    for call in (lambda: w.Lock(0), lambda: w.Unlock(0), lambda: w.GetAccumulate(x, np.zeros(4, np.int64), 0),
                 lambda: w.FetchAndOp(1, 0), lambda: w.CompareAndSwap(1, 0, 0)):
        try:
            call()
            raise AssertionError("data call succeeded without a device")
        except mpi.MpiError as e:
            if e.code != L.ERR_NO_DEVICE:
                raise
    return {"checked": 10}


W.SCENARIOS.update({k[len("scenario_"):]: v for k, v in list(globals().items()) if k.startswith("scenario_")})

if __name__ == "__main__":
    W.main()
