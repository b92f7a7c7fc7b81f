"""One rank of a test world for one-sided communication (WinCreate, Put, Get, Accumulate, Fence).
Usage as _worker.py: _rma_worker.py <scenario> --out FILE [scenario args] -mpi-* flags.  Every window
and every origin is a guarded view (_kinds_worker.Buf), and after each fence every rank checks its
whole window allocation, guards included, against the numpy model of the epoch (_rma_ref.Epoch) byte
for byte; origins are checked the same way (Put / Accumulate: unchanged, Get: the model's values)."""
import ctypes
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _footprint_worker as F  # noqa: E402
import _kinds_worker as K  # noqa: E402
import _rma_ref as R  # noqa: E402
import _worker as W  # noqa: E402
from _worker import L, mpi  # noqa: E402

DTS = {"u8": np.uint8, "f32": np.float32, "f64": np.float64, "i64": np.int64}
CODE = {"u8": L.U8, "f32": L.F32, "f64": L.F64, "i64": L.I64}
STORAGES = ("heap", "torch", "pinned", "pageable")
OPS = {"sum": L.SUM, "max": L.MAX, "min": L.MIN}
EPOCH_STRIDE = 4096


class World:
    def __init__(self):
        self.lib = L.load()
        self.rank, self.n = mpi.Rank(), mpi.Size()
        self.call = 1000

    def next_call(self):
        self.call += 1
        return self.call


def rbytes(key, nbytes):
    return np.random.default_rng([11, key]).integers(0, 256, nbytes, dtype=np.uint8)


def raw_values(dt, count, key):
    """Any bit patterns (Put and Get move bytes)."""
    return rbytes(key, count * np.dtype(dt).itemsize).view(dt)


def acc_values(dt, count, key):
    """Accumulate inputs whose sums are exact in any order (floats: integers below 2^10), full-range
    int64 (sums wrap); no NaN and no negative zero."""
    rng = np.random.default_rng([13, key])
    if np.dtype(dt) == np.int64:
        return rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, count, dtype=np.int64, endpoint=True)
    return rng.integers(-1000, 1000, count).astype(dt)


class Windows:
    """Window `key`: on every rank r `counts[r]` elements of dt at byte `offs[r]` past a heap guard
    (None: a 0-byte window at NULL), created collectively.  `images` is every rank's window as bytes."""

    def __init__(self, Wd, dt, counts, offs, key, init=None):
        self.Wd, self.dt, self.key = Wd, np.dtype(dt), key
        self.images = []
        for r in range(Wd.n):
            if counts[r] is None:
                self.images.append(np.empty(0, np.uint8))
                continue
            body = None if init is None else init(r)
            head, nbody, _, total = F.zones(counts[r], dt, offs[r])
            img = F.guard_pattern(r, key, total)[head:head + nbody].copy()
            if body is not None:
                img = np.ascontiguousarray(body, dtype=dt).view(np.uint8).copy()
            self.images.append(img)
        me = Wd.rank
        self.buf = None
        if counts[me] is not None:
            self.buf = K.Buf("heap", dt, counts[me], offs[me], me, key, body=None if init is None else init(me))
        self.win = mpi.WinCreate(self.buf.view if self.buf is not None else None)

    def check(self, images, what):
        """After a fence: this rank's window holds images[rank], the guards their pattern.  The read is
        a local access of the window, so it gets an epoch of its own: a fence after it keeps the next
        epoch's Puts and Accumulates from other ranks out until every rank has read its window."""
        self.images = images
        if self.buf is not None:
            self.buf.set_body(images[self.Wd.rank].view(self.dt))
            F.check(self.buf, what + " [window of rank %d]" % self.Wd.rank)
        self.win.Fence()

    def free(self):
        self.win.Free()
        if self.buf is not None:
            self.buf.free()


def origin_buf(Wd, storage, dt, count, key, body, off=None):
    es = np.dtype(dt).itemsize
    if off is None:
        off = (key * es) % 16 if storage != "heap" else (key * 3 * es) % 16
    return K.Buf(storage, dt, count, off, Wd.rank, key, body=body)


def do(Wd, kind, win, origin, count, code, target, disp, op=None, facade=False):
    """One Put / Get / Accumulate through the facade or the C ABI; asserts success."""
    if facade:
        view = origin.view
        if kind == "put":
            win.win.Put(view, target, disp)
        elif kind == "get":
            win.win.Get(view, target, disp)
        else:
            win.win.Accumulate(view, target, disp, op)
        return
    lib = Wd.lib
    p = origin.ptr()
    if kind == "put":
        rc = lib.b200mpi_put(p, count, code, target, disp, win.win.id, origin.memkind)
    elif kind == "get":
        rc = lib.b200mpi_get(p, count, code, target, disp, win.win.id, origin.memkind)
    else:
        rc = lib.b200mpi_accumulate(p, count, code, op, target, disp, win.win.id, origin.memkind)
    assert rc == 0, (kind, count, target, disp, rc, L.last_error())


def put_get_round(Wd, win, dn, count, i, what):
    """A Put ring shift (rank r into rank r+1) in one epoch, then a Get of the same range from every
    rank in the next; origins rotate through the storages from rank to rank."""
    rank, n = Wd.rank, Wd.n
    dt, code = DTS[dn], CODE[dn]
    disp = lambda r: (i * 5 + 3 * r) % 7  # noqa: E731  elements: misaligned mod 16 for most (r, i)
    vals = lambda r: raw_values(dt, count, 7919 * i + r)  # noqa: E731
    E = R.Epoch(win.images)
    for r in range(n):
        E.put(vals(r), (r + 1) % n, disp(r))
    storage = STORAGES[(i + rank) % 4]
    o = origin_buf(Wd, storage, dt, count, Wd.next_call(), vals(rank))
    W.trace("%s put count=%d storage=%s disp=%d" % (what, count, storage, disp(rank)))
    do(Wd, "put", win, o, count, code, (rank + 1) % n, disp(rank), facade=i % 2 == 0)
    win.win.Fence()
    F.check(o, what + " put: origin unchanged")
    o.free()
    win.check(E.fence(), what + " put")
    E = R.Epoch(win.images)
    for t in range(n):
        storage = STORAGES[(i + rank + t) % 4]
        o = origin_buf(Wd, storage, dt, count, Wd.next_call(), None)
        do(Wd, "get", win, o, count, code, t, disp(t), facade=(i + t) % 2 == 1)
        o.set_body(E.get(dt, count, t, disp(t)))
        F.check(o, what + " get from %d storage=%s" % (t, storage))
        o.free()
    win.win.Fence()
    win.check(E.fence(), what + " get: windows unchanged")
    return 1 + n


def scenario_rma(a):
    """Every dtype at counts 0, 1, 3, EPV - 1, EPV + 1, 4097 and 65537: a Put ring shift and a Get
    from every rank, at displacements mostly misaligned mod 16, into windows of a different size on
    every rank, each a sub-slice of an Alloc at a byte offset (0 on rank 0), origins from every
    storage.  Then a window that is 0 bytes at NULL on the last rank."""
    Wd = World()
    rank, n = Wd.rank, Wd.n
    done = 0
    i = 0
    for j, (dn, dt) in enumerate(DTS.items()):
        es = np.dtype(dt).itemsize
        epv = 16 // es
        counts = sorted({0, 1, 3, max(epv - 1, 0), epv + 1, 4097, 65537})
        win = Windows(Wd, dt, [65537 + 8 + 5 * r for r in range(n)], [(r * 3 * es + j) % 16 if r else 0 for r in range(n)], Wd.next_call())
        for count in counts:
            i += 1
            done += put_get_round(Wd, win, dn, count, i, "rma dtype=%s count=%d rank=%d n=%d" % (dn, count, rank, n))
        win.free()
    # the last rank's window is empty: counts 0 reach it, anything more is refused
    wcounts = [33 + r for r in range(n)]
    wcounts[n - 1] = None
    win = Windows(Wd, np.float64, wcounts, [8] * n, Wd.next_call())
    x = np.arange(4, dtype=np.float64)
    assert Wd.lib.b200mpi_put(x.ctypes.data, 0, L.F64, n - 1, 0, win.win.id, L.HOST) == 0, L.last_error()
    assert Wd.lib.b200mpi_get(x.ctypes.data, 1, L.F64, n - 1, 0, win.win.id, L.HOST) == L.ERR_ARG
    E = R.Epoch(win.images)
    t = (rank + 1) % n
    if t != n - 1:
        win.win.Put(x, t, 3)
    for r in range(n):
        if (r + 1) % n != n - 1:
            E.put(x, (r + 1) % n, 3)
    win.win.Fence()
    win.check(E.fence(), "rma with an empty window")
    win.free()
    mpi.Barrier()
    return {"checked": done + 2}


def scenario_rma_counts(a):
    """A heap Put launches exactly one kernel and leaves the heap as it was; Put, Get and Accumulate
    take no barrier epoch; each fence takes one stride (none in a world of one, where it only
    synchronises)."""
    Wd = World()
    lib, rank, n = Wd.lib, Wd.rank, Wd.n
    win = Windows(Wd, np.float32, [4096] * n, [0] * n, Wd.next_call())
    src = mpi.Alloc(1000, np.float32).copy_from_host(acc_values(np.float32, 1000, 3))
    used = ctypes.c_size_t()
    assert lib.b200mpi_heap_info(None, ctypes.byref(used), None) == 0
    used0, launches0, epoch0 = used.value, lib.b200mpi_launch_count(), L.get_param("epoch")
    win.win.Put(src, (rank + 1) % n, 17)
    assert lib.b200mpi_launch_count() == launches0 + 1, "a heap Put is one kernel"
    assert lib.b200mpi_heap_info(None, ctypes.byref(used), None) == 0 and used.value == used0, "a heap Put stages nothing"
    assert L.get_param("epoch") == epoch0, "Put takes no epoch"
    win.win.Accumulate(src, (rank + 2) % n, 1100)
    assert lib.b200mpi_launch_count() == launches0 + 2, "a heap Accumulate is one kernel"
    assert L.get_param("epoch") == epoch0, "Accumulate takes no epoch"
    win.win.Fence()
    stride = EPOCH_STRIDE if n > 1 else 0
    assert L.get_param("epoch") == epoch0 + stride, (L.get_param("epoch"), epoch0)
    dst = mpi.Alloc(1000, np.float32)
    win.win.Get(dst, (rank + 3) % n, 2000)
    assert lib.b200mpi_launch_count() == launches0 + 3 + (1 if n > 1 else 0)
    assert L.get_param("epoch") == epoch0 + stride, "Get takes no epoch"
    win.win.Fence()
    win.win.Fence()
    assert L.get_param("epoch") == epoch0 + 3 * stride
    dst.free()
    src.free()
    win.free()
    mpi.Barrier()
    return {"checked": 8}


def rule_epochs(Wd):
    """Rank 0 alone accumulates into rank 0's window, pinning the rules b200mpi.h states: the f32 SUM
    flush rule through the 16-byte red (origin and target aligned), through head, vector and tail
    (target at element 1, origin with its residue) and through the scalar red only (origin at 8 mod 16
    against an aligned target); the NaN rule of f64 MAX and f32 MIN.  Then every rank accumulates from
    a heap origin 1 to 3 bytes off its element alignment, which the library stages first."""
    rank, n = Wd.rank, Wd.n
    tiny = np.float32(R.F32_MIN_NORMAL)
    sub = np.float32(1e-39)  # subnormal
    f32_init = np.array([0.0, sub, 1.5 * tiny, -sub, -1.5 * tiny, 1.0, 2.0, -2.0], dtype=np.float32)
    f32_add = np.array([2.0 ** -140, 0.0, -tiny, 0.0, tiny, 2.0 ** -140, -sub, 3.0], dtype=np.float32)
    # hand-worked: subnormal input -> 0, subnormal result -> 0 of its sign, -0 + +0 = +0
    f32_want = np.array([0.0, 0.0, 0.0, 0.0, -0.0, 1.0, 2.0, 1.0], dtype=np.float32)
    assert np.array_equal(R.combine(f32_init, f32_add, R.SUM).view(np.uint32), f32_want.view(np.uint32))
    nan_init, nan_add = [np.nan, 1.0, -5.0, 7.0, 0.5, 2.0, -1.0, 9.0], [3.0, np.nan, -6.0, 7.5, 0.25, 4.0, -2.0, np.nan]
    done = 0
    for dt, init, add, op, disp, off in ((np.float32, f32_init, f32_add, R.SUM, 0, 0),
                                         (np.float32, f32_init, f32_add, R.SUM, 1, 4),
                                         (np.float32, f32_init, f32_add, R.SUM, 0, 8),
                                         (np.float64, nan_init, nan_add, R.MAX, 1, 8),
                                         (np.float32, nan_init, nan_add, R.MIN, 0, 4)):
        init, add = np.array(init, dtype=dt), np.array(add, dtype=dt)
        body = np.zeros(len(init) + 1, dtype=dt)
        body[disp:disp + len(init)] = init
        win = Windows(Wd, dt, [len(body)] * n, [0] * n, Wd.next_call(), init=lambda r: body)
        E = R.Epoch(win.images)
        E.accumulate(add, 0, disp, op)
        if rank == 0:
            o = origin_buf(Wd, "heap", dt, len(add), 99, add, off=off)
            do(Wd, "acc", win, o, len(add), L.F32 if dt == np.float32 else L.F64, 0, disp, op)
            F.check(o, "rule epoch: origin unchanged")
            o.free()
            if op == R.SUM:
                assert np.array_equal(E.now[0].view(np.uint32)[disp:disp + len(add)], f32_want.view(np.uint32))
        win.win.Fence()
        win.check(E.fence(), "rule epoch dtype=%s op=%d disp=%d origin residue=%d" % (np.dtype(dt), op, disp, off))
        win.free()
        done += 1
    # heap origins off their element alignment
    win = Windows(Wd, np.float32, [300] * n, [4] * n, Wd.next_call(), init=lambda r: acc_values(np.float32, 300, 77 + r))
    E = R.Epoch(win.images)
    for r in range(n):
        E.accumulate(acc_values(np.float32, 257, 88 + r), (r + 1) % n, 5, R.SUM)
    o = origin_buf(Wd, "heap", np.float32, 257, Wd.next_call(), acc_values(np.float32, 257, 88 + rank), off=1 + rank % 3)
    do(Wd, "acc", win, o, 257, L.F32, (rank + 1) % n, 5, R.SUM, facade=rank % 2 == 1)
    F.check(o, "misaligned heap origin unchanged")
    o.free()
    win.win.Fence()
    win.check(E.fence(), "accumulate from a heap origin off its element alignment")
    win.free()
    return done + 1


def scenario_rma_accumulate(a):
    """Every rank accumulates into overlapping ranges of rank 0's window and of every rank's window,
    several calls per epoch, for f32, f64 and i64 with SUM, MAX and MIN (each op in its own epoch on the
    same window), origins from every storage, at origin residues that agree with the target mod 16
    (vector path) and that do not.  Then rule_epochs."""
    Wd = World()
    rank, n = Wd.rank, Wd.n
    done = 0
    i = 0
    for dn in ("f32", "f64", "i64"):
        dt, code = DTS[dn], CODE[dn]
        es = np.dtype(dt).itemsize
        M = 9000
        key = Wd.next_call()
        win = Windows(Wd, dt, [M + 11 * r for r in range(n)], [(es * r) % 16 for r in range(n)], key,
                      init=lambda r: acc_values(dt, M + 11 * r, key * 10 + r))
        for opname, op in OPS.items():
            E = R.Epoch(win.images)
            calls = []  # (rank, target, disp, count, values key)
            for r in range(n):
                for k, (t, count) in enumerate(((0, 4099), (r, 3), (0, 1), ((r + 1) % n, 2000))):
                    disp = 7 * r + 3 * k if t == 0 else 5 * k + r
                    calls.append((r, t, disp, count, 100000 * i + 100 * r + k))
            for _ in range(2):  # the same calls twice: several Accumulates per location and epoch
                for r, t, disp, count, vk in calls:
                    E.accumulate(acc_values(dt, count, vk), t, disp, op)
            for rep in range(2):
                for r, t, disp, count, vk in calls:
                    if r != rank:
                        continue
                    i += 1
                    storage = STORAGES[(i + rank) % 4]
                    agree = (i % 2 == 0)
                    tgt_res = (((es * t) % 16) + disp * es) % 16
                    off = tgt_res if agree or storage != "heap" else (tgt_res + es) % 16
                    o = origin_buf(Wd, storage, dt, count, Wd.next_call(), acc_values(dt, count, vk), off=off)
                    do(Wd, "acc", win, o, count, code, t, disp, op, facade=i % 3 == 0)
                    F.check(o, "accumulate origin unchanged")
                    o.free()
            win.win.Fence()
            win.check(E.fence(), "accumulate dtype=%s op=%s rank=%d n=%d" % (dn, opname, rank, n))
            done += 1
        win.free()
    done += rule_epochs(Wd)
    mpi.Barrier()
    return {"checked": done}


def scenario_rma_epochs(a):
    """Several consecutive epochs on one window, with collectives on other buffers issued between the
    RMA calls and the fence (an Allreduce, a Bcast, a Barrier), and each fence taking one stride."""
    Wd = World()
    rank, n = Wd.rank, Wd.n
    dt = np.int64
    M = 3000
    key = Wd.next_call()
    win = Windows(Wd, dt, [M] * n, [8] * n, key, init=lambda r: acc_values(dt, M, key + r))
    x = mpi.Alloc(513, np.int64)
    done = 0
    for e in range(6):
        E = R.Epoch(win.images)
        for r in range(n):
            E.put(acc_values(dt, 100, 50 * e + r), (r + e + 1) % n, 10 * r)
            E.accumulate(acc_values(dt, 300, 70 * e + r), (r + e) % n, 1000 + 7 * r, R.SUM)
        win.win.Put(acc_values(dt, 100, 50 * e + rank), (rank + e + 1) % n, 10 * rank)
        x.copy_from_host(np.full(513, rank + e, dtype=np.int64))
        mpi.Allreduce(x, x)
        assert np.array_equal(x.to_host(), np.full(513, sum(r + e for r in range(n)), dtype=np.int64)), "allreduce between RMA calls"
        win.win.Accumulate(acc_values(dt, 300, 70 * e + rank), (rank + e) % n, 1000 + 7 * rank)
        b = np.full(17, rank, dtype=np.int64)
        mpi.Bcast(b, e % n)
        assert np.array_equal(b, np.full(17, e % n)), "bcast between RMA calls"
        mpi.Barrier()
        epoch0 = L.get_param("epoch")
        win.win.Fence()
        assert L.get_param("epoch") == epoch0 + (EPOCH_STRIDE if n > 1 else 0)
        win.check(E.fence(), "epoch %d" % e)
        done += 1
    x.free()
    win.free()
    mpi.Barrier()
    return {"checked": done}


def scenario_rma_capped(a):
    """Grids capped at 1 and 3 CTAs: every Put, Get and Accumulate makes several grid passes.  The
    Accumulate comes first, while the window holds integer values (a Put writes any bit pattern)."""
    Wd = World()
    rank, n = Wd.rank, Wd.n
    done = 0
    for cap in (1, 3):
        assert Wd.lib.b200mpi_set_max_blocks(cap) == 0
        for dn in ("f32", "f64", "u8"):
            dt = DTS[dn]
            count = 300007 if dn != "u8" else 1000003
            key = Wd.next_call()
            win = Windows(Wd, dt, [count + 16] * n, [(8 * r) % 16 for r in range(n)], key,
                          init=(lambda r: acc_values(dt, count + 16, key + r)) if dn != "u8" else None)
            if dn != "u8":
                E = R.Epoch(win.images)
                for r in range(n):
                    E.accumulate(acc_values(dt, count, 9 + r), (r + 1) % n, 4, R.SUM)
                o = origin_buf(Wd, "heap", dt, count, Wd.next_call(), acc_values(dt, count, 9 + rank), off=(8 * ((rank + 1) % n) + 4 * np.dtype(dt).itemsize) % 16)
                do(Wd, "acc", win, o, count, CODE[dn], (rank + 1) % n, 4, R.SUM)
                o.free()
                win.win.Fence()
                win.check(E.fence(), "capped=%d accumulate %s" % (cap, dn))
                done += 1
            done += put_get_round(Wd, win, dn, count, cap + len(dn), "capped=%d dtype=%s" % (cap, dn))
            win.free()
    assert Wd.lib.b200mpi_set_max_blocks(0) == 0
    mpi.Barrier()
    return {"checked": done}


def scenario_rma_errors(a):
    """Every argument error returns its code and writes nothing (every window is checked after a
    fence); windows that ranks refuse to create are created nowhere, and the next id still agrees."""
    Wd = World()
    lib, rank, n = Wd.lib, Wd.rank, Wd.n
    key = Wd.next_call()
    win = Windows(Wd, np.float64, [64 + r for r in range(n)], [0] * n, key)
    odd = Windows(Wd, np.uint8, [256] * n, [3] * n, Wd.next_call())  # window base 3 bytes into a heap block
    wid = win.win.id
    a8 = mpi.Alloc(64, np.float64)
    p = a8.ptr
    h = np.zeros(64, dtype=np.float64)
    hp = h.ctypes.data
    big = (1 << 64) - 1
    t = (rank + 1) % n
    cases = (
        ("unknown window put", lambda: lib.b200mpi_put(p, 1, L.F64, t, 0, wid + 100, L.DEVICE), L.ERR_ARG),
        ("negative window get", lambda: lib.b200mpi_get(p, 1, L.F64, t, 0, -1, L.DEVICE), L.ERR_ARG),
        ("unknown window fence", lambda: lib.b200mpi_win_fence(wid + 100), L.ERR_ARG),
        ("unknown window free", lambda: lib.b200mpi_win_free(-3), L.ERR_ARG),
        ("unknown dtype put", lambda: lib.b200mpi_put(p, 1, 9, t, 0, wid, L.DEVICE), L.ERR_ARG),
        ("unknown dtype accumulate", lambda: lib.b200mpi_accumulate(p, 1, 9, L.SUM, t, 0, wid, L.DEVICE), L.ERR_ARG),
        ("u8 accumulate", lambda: lib.b200mpi_accumulate(p, 1, L.U8, L.SUM, t, 0, wid, L.DEVICE), L.ERR_UNSUPPORTED),
        ("unknown op", lambda: lib.b200mpi_accumulate(p, 1, L.F64, 7, t, 0, wid, L.DEVICE), L.ERR_ARG),
        ("target = size", lambda: lib.b200mpi_put(p, 1, L.F64, n, 0, wid, L.DEVICE), L.ERR_ARG),
        ("negative target", lambda: lib.b200mpi_accumulate(p, 1, L.I64, L.MAX, -1, 0, wid, L.DEVICE), L.ERR_ARG),
        ("bad memkind", lambda: lib.b200mpi_get(p, 1, L.F64, t, 0, wid, 5), L.ERR_ARG),
        ("NULL origin put", lambda: lib.b200mpi_put(None, 1, L.F64, t, 0, wid, L.HOST), L.ERR_ARG),
        ("NULL origin get", lambda: lib.b200mpi_get(None, 2, L.F64, t, 0, wid, L.DEVICE), L.ERR_ARG),
        ("past the window by one", lambda: lib.b200mpi_put(hp, 2, L.F64, t, 64 + t - 1, wid, L.HOST), L.ERR_ARG),
        ("count past the window", lambda: lib.b200mpi_get(hp, 65 + t, L.F64, t, 0, wid, L.HOST), L.ERR_ARG),
        ("displacement overflow", lambda: lib.b200mpi_put(hp, 2, L.F64, t, big, wid, L.HOST), L.ERR_ARG),
        ("displacement times size overflow", lambda: lib.b200mpi_accumulate(hp, 1, L.F64, L.SUM, t, big // 8 + 1, wid, L.HOST), L.ERR_ARG),
        ("misaligned accumulate target", lambda: lib.b200mpi_accumulate(hp, 1, L.F32, L.SUM, t, 0, odd.win.id, L.HOST), L.ERR_ARG),
        ("misaligned accumulate target i64", lambda: lib.b200mpi_accumulate(hp, 2, L.I64, L.MIN, t, 1, odd.win.id, L.HOST), L.ERR_ARG),
    )
    done = 0
    for name, call, want in cases:
        rc = call()
        assert rc == want, (name, rc, want, L.last_error())
        done += 1
    # legal corner cases: count 0 with NULL or huge displacements, the exact fit
    assert lib.b200mpi_put(None, 0, L.F64, t, big, wid, L.HOST) == 0, L.last_error()
    assert lib.b200mpi_accumulate(None, 0, L.F64, L.SUM, t, 0, wid, L.DEVICE) == 0, L.last_error()
    E = R.Epoch(win.images)
    fit = np.arange(2, dtype=np.float64) + rank
    assert lib.b200mpi_put(fit.ctypes.data, 2, L.F64, t, 64 + t - 2, wid, L.HOST) == 0, L.last_error()
    for r in range(n):
        E.put(np.arange(2, dtype=np.float64) + r, (r + 1) % n, 64 + (r + 1) % n - 2)
    win.win.Fence()
    odd.win.Fence()
    win.check(E.fence(), "errors: only the exact fit was written")
    odd.check(odd.images, "errors: the odd window is untouched")
    done += 2
    wide = Windows(Wd, np.uint8, [0] * n, [0] * n, Wd.next_call())  # a 0-byte window on every rank
    assert lib.b200mpi_put(fit.ctypes.data, 1, L.U8, t, 0, wide.win.id, L.HOST) == L.ERR_ARG, L.last_error()
    # win_create refusals: rank 0 passes host memory; then every rank a NULL base with bytes
    wid_before = win.win.id
    wc = ctypes.c_int(-7)
    rc = lib.b200mpi_win_create(hp if rank == 0 else a8.ptr, 64, ctypes.byref(wc))
    assert rc == (L.ERR_ARG if rank == 0 else L.ERR_PEER) and wc.value == -7, (rc, wc.value, L.last_error())
    rc = lib.b200mpi_win_create(None, 16, ctypes.byref(wc))
    assert rc == L.ERR_ARG and wc.value == -7, (rc, L.last_error())
    rc = lib.b200mpi_win_create(a8.ptr, 16, None)
    assert rc == L.ERR_ARG, (rc, L.last_error())
    wc2 = ctypes.c_int(-1)
    assert lib.b200mpi_win_create(a8.ptr, 16, ctypes.byref(wc2)) == 0, L.last_error()
    assert wc2.value == wide.win.id + 1 and wc2.value > wid_before, (wc2.value, wide.win.id)
    assert lib.b200mpi_win_free(wc2.value) == 0, L.last_error()
    assert lib.b200mpi_put(fit.ctypes.data, 1, L.F64, t, 0, wc2.value, L.HOST) == L.ERR_ARG, "freed window"
    assert lib.b200mpi_win_fence(wc2.value) == L.ERR_ARG and lib.b200mpi_win_free(wc2.value) == L.ERR_ARG
    done += 6
    wide.free()
    odd.free()
    win.free()
    a8.free()
    mpi.Barrier()
    return {"checked": done}


def scenario_rma_nomem(a):
    """A host origin whose staging block does not fit in the heap: B200MPI_ERR_NOMEM from Put and Get,
    with the window and the origin untouched."""
    Wd = World()
    lib, rank, n = Wd.lib, Wd.rank, Wd.n
    total, used = ctypes.c_size_t(), ctypes.c_size_t()
    assert lib.b200mpi_heap_info(ctypes.byref(total), ctypes.byref(used), None) == 0
    count = (total.value - used.value) * 2 // 3  # the window leaves less than this free for staging
    wmem = mpi.Alloc(count, np.uint8).copy_from_host(np.full(count, 7, dtype=np.uint8))
    w = mpi.WinCreate(wmem)
    hog = np.ones(count, dtype=np.uint8)
    t = (rank + 1) % n
    for call in (lambda: lib.b200mpi_put(hog.ctypes.data, count, L.U8, t, 0, w.id, L.HOST),
                 lambda: lib.b200mpi_get(hog.ctypes.data, count, L.U8, t, 0, w.id, L.HOST)):
        rc = call()
        assert rc == L.ERR_NOMEM, (rc, L.last_error())
    assert np.all(hog == 1), "get wrote the origin"
    w.Fence()
    assert np.all(wmem.to_host() == 7), "nomem: the window was written"
    w.Free()
    wmem.free()
    mpi.Barrier()
    return {"checked": 2}


def scenario_rma_mismatch(a):
    """Fences on different windows, and a fence against a Barrier, end as B200MPI_ERR_PEER on every
    rank with no window touched; the next fence works."""
    Wd = World()
    rank, n = Wd.rank, Wd.n
    A = Windows(Wd, np.float32, [100] * n, [0] * n, Wd.next_call())
    B = Windows(Wd, np.float32, [100] * n, [4] * n, Wd.next_call())
    lib = Wd.lib
    rc = lib.b200mpi_win_fence(B.win.id if rank == 1 else A.win.id)
    assert rc == L.ERR_PEER, (rc, L.last_error())
    rc = lib.b200mpi_win_fence(A.win.id) if rank == 0 else lib.b200mpi_barrier()
    assert rc == L.ERR_PEER, (rc, L.last_error())
    rc = lib.b200mpi_win_free(A.win.id) if rank == n - 1 else lib.b200mpi_win_fence(B.win.id)
    assert rc == L.ERR_PEER, (rc, L.last_error())
    E = R.Epoch(A.images)
    x = np.full(10, rank + 0.5, dtype=np.float32)
    A.win.Put(x, (rank + 1) % n, 50)
    for r in range(n):
        E.put(np.full(10, r + 0.5, dtype=np.float32), (r + 1) % n, 50)
    A.win.Fence()
    A.check(E.fence(), "mismatch: the next fence works")
    B.win.Fence()
    B.check(B.images, "mismatch: B untouched")
    A.free()
    B.free()
    mpi.Barrier()
    return {"checked": 4}


def scenario_rma_large(a):
    """64 MiB per rank: a Put ring shift of f32, a Get of the whole neighbour window, and f64 SUM
    Accumulates from every rank into rank 0, checked against numpy."""
    Wd = World()
    rank, n = Wd.rank, Wd.n
    nb = 64 << 20
    win = mpi.Alloc(nb // 4, np.float32)
    win.copy_from_host(np.zeros(nb // 4, dtype=np.float32))
    w = mpi.WinCreate(win)
    vals = lambda r: acc_values(np.float32, nb // 4, 500 + r)  # noqa: E731
    src = mpi.Alloc(nb // 4, np.float32).copy_from_host(vals(rank))
    w.Put(src, (rank + 1) % n, 0)
    w.Fence()
    W.check_equal(win.to_host(), vals((rank - 1) % n), "large put")
    got = np.empty(nb // 4, dtype=np.float32)
    w.Get(got, (rank + 1) % n, 0)
    W.check_equal(got, vals(rank), "large get")
    w.Fence()
    w.Free()
    dwin = mpi.DeviceSlice(nb // 8, np.float64, win.ptr, owner=False)
    dwin.copy_from_host(np.zeros(nb // 8))
    w = mpi.WinCreate(dwin)
    dv = lambda r: acc_values(np.float64, nb // 8, 900 + r)  # noqa: E731
    dsrc = mpi.DeviceSlice(nb // 8, np.float64, src.ptr, owner=False).copy_from_host(dv(rank))
    w.Accumulate(dsrc, 0, 0)
    w.Fence()
    if rank == 0:
        W.check_equal(dwin.to_host(), np.sum([dv(r) for r in range(n)], axis=0), "large accumulate")
    w.Free()
    src.free()
    win.free()
    mpi.Barrier()
    return {"checked": 3}


def scenario_rma_control_only(a):
    """Control plane only: all six entries refuse with B200MPI_ERR_NO_DEVICE, through the C ABI and the facade."""
    lib = L.load()
    x = np.zeros(4, np.float64)
    wc = ctypes.c_int(-1)
    assert lib.b200mpi_win_create(None, 0, ctypes.byref(wc)) == L.ERR_NO_DEVICE
    assert lib.b200mpi_win_free(0) == L.ERR_NO_DEVICE
    assert lib.b200mpi_win_fence(0) == L.ERR_NO_DEVICE
    assert lib.b200mpi_put(x.ctypes.data, 4, L.F64, 0, 0, 0, L.HOST) == L.ERR_NO_DEVICE
    assert lib.b200mpi_get(x.ctypes.data, 4, L.F64, 0, 0, 0, L.HOST) == L.ERR_NO_DEVICE
    assert lib.b200mpi_accumulate(x.ctypes.data, 4, L.F64, L.SUM, 0, 0, 0, L.HOST) == L.ERR_NO_DEVICE
    w = mpi.Win(0)
    for call in (lambda: mpi.WinCreate(None), lambda: w.Put(x, 0), lambda: w.Get(x, 0), lambda: w.Accumulate(x, 0),
                 w.Fence, w.Free):
        try:
            call()
            raise AssertionError("data call succeeded without a device")
        except mpi.MpiError as e:
            if e.code != L.ERR_NO_DEVICE:
                raise
    return {"checked": 12}


W.SCENARIOS.update({k[len("scenario_"):]: v for k, v in list(globals().items()) if k.startswith("scenario_")})

if __name__ == "__main__":
    W.main()
