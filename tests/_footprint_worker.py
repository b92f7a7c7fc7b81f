"""One rank of a test world that checks what every collective writes, and what it must leave alone.
Usage as _worker.py: _footprint_worker.py footprint --out FILE [--parts ...] -mpi-* flags.

Every buffer a rank passes is a view into a larger allocation with GUARD bytes on each side, at a
byte offset picked per call from four layouts (all 16-byte aligned, the same misalignment on every
rank, a different residue mod 16 per rank, send and recv misaligned differently).  The guards and
every byte the call must not write hold a pattern no kernel produces.  After each call every rank
compares the whole allocation of every buffer it passed with what it must hold: the guards and an
out-of-place send unchanged, the destination equal to the oracle in the order of the kernel that
ran.  The reductions see signed values over a wide exponent range with +-0, +-Inf, NaN, subnormals
and +-max (INT64_MIN/MAX, -1 and 0 for i64) at rank-dependent positions, so MAX and MIN results
depend on each kernel's order and are compared bit for bit."""
import argparse
import ctypes
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _alltoallv_ref as AV  # noqa: E402
import _gather_oracle as G  # noqa: E402
import _worker as W  # noqa: E402
from _gather_worker import v_tables  # noqa: E402
from _worker import ALGOS, L, O, SEED, expect_allreduce, mpi  # noqa: E402

GUARD = 64
LAYOUTS = ("aligned", "symmetric", "mixed", "split")
DTYPES = {"u8": np.uint8, "f32": np.float32, "f64": np.float64, "i64": np.int64}
OPS = (("sum", mpi.SUM, O.SUM), ("max", mpi.MAX, O.MAX), ("min", mpi.MIN, O.MIN))
# byte residues mod 16 a view of each element type can start at; the order of the u8 list mixes
# access widths (16, 8, 4 and 1 byte) between neighbouring ranks
RESIDUES = {np.dtype(np.uint8): (0, 8, 4, 1, 12, 2, 7, 15, 3, 5, 6, 9, 10, 11, 13, 14),
            np.dtype(np.float32): (0, 8, 4, 12), np.dtype(np.float64): (0, 8), np.dtype(np.int64): (0, 8)}
NOT_WRITTEN = (0x00, 0xFF, 0xA5)  # byte values a kernel plausibly leaves (zeroing, -1 fills, old sentinels)


def epv(dt):
    return 16 // np.dtype(dt).itemsize


def guard_pattern(rank, call, nbytes):
    """Bytes 0x41..0x7D in a sequence that depends on rank and call: never 0x00, 0xFF or 0xA5."""
    i = np.arange(nbytes, dtype=np.int64)
    return (0x41 + (i * 7 + rank * 13 + call * 29) % 0x3D).astype(np.uint8)


def zones(count, dt, off):
    """(head, body, tail, total) byte lengths of the allocation behind a view of `count` elements
    that starts `off` bytes past the GUARD-byte head guard.  The tail guard is GUARD bytes or more,
    so that the whole allocation is a multiple of 16 bytes."""
    head = GUARD + off
    body = count * np.dtype(dt).itemsize
    tail = GUARD + (-(head + body)) % 16
    return head, body, tail, head + body + tail


def layout_offsets(layout, dt, n, key):
    """[(send_off, recv_off)] byte offsets from the guard for every rank; the same on every rank for
    the same key.  A random multiple of 16 is added so that views move within the heap."""
    res = RESIDUES[np.dtype(dt)]
    rng = np.random.default_rng([SEED, key])
    lift = [16 * int(x) for x in rng.integers(0, 3, size=2 * n)]
    if layout == "aligned":
        return [(lift[2 * r], lift[2 * r + 1]) for r in range(n)]
    if layout == "symmetric":
        m = res[1 + int(rng.integers(len(res) - 1))] + lift[0]
        return [(m, m)] * n
    if layout == "mixed":
        s = int(rng.integers(len(res)))
        return [(res[(s + r) % len(res)] + lift[2 * r], res[(s + r) % len(res)] + lift[2 * r + 1]) for r in range(n)]
    if layout == "split":
        out = []
        for r in range(n):
            a, b = rng.choice(len(res), size=2, replace=False)
            out.append((res[a] + lift[2 * r], res[b] + lift[2 * r + 1]))
        return out
    raise ValueError(layout)


# ---- values ------------------------------------------------------------------------------------
def _qnan(dt, payload):
    if np.dtype(dt) == np.float32:
        return np.array([0x7FC00000 | payload], dtype=np.uint32).view(np.float32)[0]
    return np.array([0x7FF8000000000000 | payload], dtype=np.uint64).view(np.float64)[0]


def specials(dt, rank):
    """The values whose MAX / MIN depend on the order of the operands, or that overflow a SUM.  The
    NaN payload names the rank it came from, so a result shows whose NaN went through."""
    dt = np.dtype(dt)
    if dt == np.int64:
        return np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, -1, 0], dtype=np.int64)
    fi = np.finfo(dt)
    sub = fi.smallest_subnormal
    return np.array([0.0, -0.0, np.inf, -np.inf, _qnan(dt, 0x100 + rank), sub, -sub, fi.tiny / 3, -fi.tiny / 3, fi.max, -fi.max], dtype=dt)


def special_slots(dt, n, count):
    """[(special index, position, rank)]: every special at a position where rank 0 holds it (first
    in rank order), one where a middle rank holds it and one where rank n-1 holds it, the positions
    spread over the whole message."""
    m = len(specials(dt, 0))
    slots = []
    for k in range(m):
        for j, who in enumerate((0, n // 2, n - 1)):
            t = 3 * k + j
            p = t * count // (3 * m) if count >= 3 * m else t
            if p < count:
                slots.append((k, p, who))
    return slots


def gen_values(dt, n, count, seed):
    """Every rank's input of one call.  u8: random bytes.  Floats: random sign and mantissa, exponents
    over a wide range; a quarter of the positions are clashes where each rank holds +0, -0, its NaN,
    +-Inf or a plain value, so that NaN and signed zeros meet in every order; then the special_slots.
    i64: the full range, clashes of INT64_MIN / INT64_MAX / -1 / 0."""
    dt = np.dtype(dt)
    rng = np.random.default_rng([SEED, seed])
    if dt == np.uint8:
        return [rng.integers(0, 256, size=count, dtype=np.uint8) for _ in range(n)]
    if dt == np.int64:
        xs = [rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, size=count, dtype=np.int64, endpoint=True) for _ in range(n)]
    else:
        emax = 30 if dt == np.float32 else 100
        xs = []
        for _ in range(n):
            mant = rng.uniform(1.0, 2.0, size=count) * rng.choice([-1.0, 1.0], size=count)
            xs.append(np.ldexp(mant, rng.integers(-emax, emax + 1, size=count)).astype(dt))
    clash = np.flatnonzero(rng.random(count) < 0.25)
    for r in range(n):
        sp = specials(dt, r)
        pool = sp[:5] if dt != np.int64 else sp  # floats: +0, -0, +Inf, -Inf, NaN
        pick = rng.integers(0, len(pool) + 2, size=clash.size)  # two extra slots: keep the plain value
        sel = pick < len(pool)
        xs[r][clash[sel]] = pool[pick[sel]]
    for k, p, who in special_slots(dt, n, count):
        xs[who][p] = specials(dt, who)[k]
    return xs


# ---- guarded buffers ---------------------------------------------------------------------------
class Guarded:
    """`count` elements of `dt` at byte `off` past the head guard of a larger allocation: a heap
    DeviceSlice or an aligned host numpy view.  `image` is what the whole allocation must hold."""

    def __init__(self, kind, dt, count, off, rank, call, body=None):
        self.kind, self.dt, self.count, self.off = kind, np.dtype(dt), int(count), int(off)
        self.head, self.nbody, self.tail, self.total = zones(count, dt, off)
        self.image = guard_pattern(rank, call, self.total)
        if body is not None:
            self.set_body(body)
        if kind == "heap":
            self.mem = self.alloc(self.total).copy_from_host(self.image)
            self.view = mpi.DeviceSlice(self.count, self.dt, self.mem.ptr + self.head, owner=False)
        else:
            raw = np.empty(self.total + 64, dtype=np.uint8)
            s = (-raw.ctypes.data) % 64
            self.mem = raw[s:s + self.total]
            self.mem[:] = self.image
            self.view = self.mem[self.head:self.head + self.nbody].view(self.dt)

    def alloc(self, nbytes):
        """The heap allocation behind a 'heap' buffer."""
        return mpi.Alloc(nbytes, np.uint8)

    def set_body(self, arr, lo=0):
        """The elements from `lo` on must hold `arr` after the call."""
        b = np.ascontiguousarray(arr, dtype=self.dt).view(np.uint8)
        a = self.head + lo * self.dt.itemsize
        self.image[a:a + b.size] = b

    def body(self, image=None):
        src = self.image if image is None else image
        return src[self.head:self.head + self.nbody].view(self.dt)

    def load(self):
        """Write the image into the allocation (after set_body on an existing buffer)."""
        if self.kind == "heap":
            self.mem.copy_from_host(self.image)
        else:
            self.mem[:] = self.image

    def sub(self, lo, hi):
        if self.kind == "heap":
            return mpi.DeviceSlice(hi - lo, self.dt, self.view.ptr + lo * self.dt.itemsize, owner=False)
        return self.view[lo:hi]

    def ptr(self):
        if self.kind == "heap":
            return self.view.ptr
        return self.view.ctypes.data if self.count else None

    def read(self):
        return self.mem.to_host() if self.kind == "heap" else np.array(self.mem, copy=True)

    def free(self):
        if self.kind == "heap":
            self.mem.free()


def where(g, i):
    """'<side> byte <k>' for byte i of g's allocation."""
    if i < g.head:
        return "head guard byte %d of %d" % (i, g.head)
    if i < g.head + g.nbody:
        k = i - g.head
        return "body byte %d (element %d)" % (k, k // g.dt.itemsize)
    return "tail guard byte %d of %d" % (i - g.head - g.nbody, g.tail)


def first_diff(g, got, want, what):
    bad = np.flatnonzero(got != want)
    if bad.size:
        i = int(bad[0])
        raise AssertionError("%s: first differing byte at %s: got 0x%02x want 0x%02x (%d bytes differ)" % (what, where(g, i), got[i], want[i], bad.size))


def check(g, what, mode="exact", ins=None, lo=0):
    """The whole allocation against g.image.  mode 'exact': every byte.  'sum' and 'tol' apply to the
    reduced elements only: the len(ins[0]) elements from element `lo` of the body (the whole body from
    `lo` without `ins`); every other byte, guards included, must match exactly.  'sum': NaN positions
    must agree and every other reduced element bit for bit.  'tol': NaN positions as for 'sum', finite
    elements within 1e-6 * sum_r |x_r| (the switch reduces in its own order)."""
    got = g.read()
    if mode == "exact" or g.dt.kind != "f":
        first_diff(g, got, g.image, what)
        return
    es = g.dt.itemsize
    k = g.count - lo if ins is None else len(ins[0])
    a, b = g.head + lo * es, g.head + (lo + k) * es
    outside = got.copy()
    outside[a:b] = g.image[a:b]
    first_diff(g, outside, g.image, what)
    gv, wv = got[a:b].view(g.dt), g.image[a:b].view(g.dt)
    nan_g, nan_w = np.isnan(gv), np.isnan(wv)
    if not np.array_equal(nan_g, nan_w):
        i = int(np.flatnonzero(nan_g != nan_w)[0])
        raise AssertionError("%s: NaN pattern differs first at %s: got %r want %r" % (what, where(g, a + i * es), gv[i], wv[i]))
    if mode == "sum" or ins is None:
        gb, wb = got.copy(), g.image.copy()
        gb[a:b][np.repeat(nan_w, es)] = 0
        wb[a:b][np.repeat(nan_w, es)] = 0
        first_diff(g, gb, wb, what)
        return
    with np.errstate(invalid="ignore", over="ignore"):
        scale = np.sum([np.abs(np.asarray(x, dtype=np.float64)) for x in ins], axis=0)
        err = np.abs(gv.astype(np.float64) - wv.astype(np.float64))
        ok = nan_w | (gv == wv) | (np.isfinite(wv) & (err <= 1e-6 * scale + 1e-300))
    if not np.all(ok):
        i = int(np.flatnonzero(~ok)[0])
        raise AssertionError("%s: %s got %r want %r (tolerance 1e-6 * %g)" % (what, where(g, a + i * es), gv[i], wv[i], scale[i]))


# ---- the run -----------------------------------------------------------------------------------
class Run:
    def __init__(self, a):
        self.lib = L.load()
        self.rank, self.n = mpi.Rank(), mpi.Size()
        info = (ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int())
        self.lib.b200mpi_heap_info(ctypes.byref(info[0]), ctypes.byref(info[1]), ctypes.byref(info[2]))
        self.nvls = bool(info[2].value)
        self.call = 0
        self.done = {}
        self.skipped = set()
        self.trim = a.trim
        self.pipe_min = L.get_param("pipe_min_bytes")

    def next_call(self, part):
        self.call += 1
        self.done[part] = self.done.get(part, 0) + 1
        return self.call

    def what(self, coll, algo, dt, opname, count, layout, offs, kind, inplace=False, root=None):
        s = "%s algo=%s dtype=%s op=%s count=%d kind=%s layout=%s inplace=%s" % (
            coll, L.ALGO_NAMES.get(algo, algo), np.dtype(dt).name, opname, count, kind, layout, inplace)
        if root is not None:
            s += " root=%d" % root
        return s + " offsets(send,recv) per rank=%s rank=%d" % (offs, self.rank)

    def kind_for(self, i, nbytes):
        """One call in four uses host views (staged copies), as long as it stays below the chunked pipeline."""
        return "host" if i % 4 == 3 and nbytes < self.pipe_min else "heap"


def counts_for(dt, passes, trim="full"):
    """0, 1, EPV-1, EPV+1, 257, 4097 and one grid pass +-1 vector of the kernel under test (`passes`
    in vectors; one-shot has one per form).  trim 'lean': without EPV-1 and 257; 'edges': 1, EPV+1 and
    the passes."""
    e = epv(dt)
    base = {"full": [0, 1, e - 1, e + 1, 257, 4097], "lean": [0, 1, e + 1, 4097], "edges": [1, e + 1]}[trim]
    for p in passes:
        base += [p * e - e, p * e + e]
    out = []
    for c in base:
        if c >= 0 and c not in out:
            out.append(c)
    return out


def mode_for(opname, dt, order):
    if opname != "sum" or np.dtype(dt) == np.int64:
        return "exact"
    return "tol" if order == O.ORDER_F64 else "sum"


def allreduce_passes(algo, n, dt):
    """Vectors per rank-world message at which the kernel's grid gains a CTA (b200mpi.cu's grid rules)."""
    pow2 = n in (2, 4, 8)
    if algo == "oneshot":  # the shuffle form sizes its grid by n lanes per vector; above 4096 vectors the rank-order form
        return [512 // n, 9 * 512] if pow2 else [512]
    if algo == "twoshot":
        u = (8 if np.dtype(dt).itemsize == 4 else 4) if n == 2 else 4 if n == 4 else 2 if n == 8 else 1
        return [n * 512 * u]
    if algo == "smem":
        return [n * 256]  # one 4 KiB tile per rank
    if algo == "ring":
        return [n * 512 * 4]
    if algo == "ll":
        return [256 * 8 // 16]  # one 8-byte cell per thread of a 256-thread CTA
    raise ValueError(algo)


def do_allreduce(R, algo, dn, count, layout, opname, inplace, kind, coll="allreduce"):
    lib, rank, n = R.lib, R.rank, R.n
    dt = DTYPES[dn]
    op, oop = {o[0]: (o[1], o[2]) for o in OPS}[opname]
    call = R.next_call(coll)
    offs = layout_offsets(layout, dt, n, call)
    if inplace:
        offs = [(s, s) for s, _ in offs]
    ins = gen_values(dt, n, count, call)
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS[algo])
    used = lib.b200mpi_get_algo(L.COLL_ALLREDUCE, count, O.NP2DT[np.dtype(dt)])
    send = Guarded(kind, dt, count, offs[rank][0], rank, call, body=ins[rank])
    recv = send if inplace else Guarded(kind, dt, count, offs[rank][1], rank, call + 1)
    mpi.Allreduce(send.view, recv.view, op)
    want, order = expect_allreduce(ins, oop, used, n, count, dt)
    what = R.what(coll, used, dt, opname, count, layout, offs, kind, inplace)
    recv.set_body(want)
    check(recv, what + " [recv]", mode_for(opname, dt, order), ins)
    if not inplace:
        check(send, what + " [send must be unchanged]")
        recv.free()
    send.free()


def part_allreduce(R):
    n = R.n
    for algo in ("oneshot", "twoshot", "smem", "ring", "ll"):
        for di, dn in enumerate(("f32", "f64", "i64")):
            dt = DTYPES[dn]
            for ci, count in enumerate(counts_for(dt, allreduce_passes(algo, n, dt), R.trim)):
                for li, layout in enumerate(LAYOUTS):
                    i = ci + li + di
                    inplace = layout in ("aligned", "mixed") and ci % 2 == 1
                    do_allreduce(R, algo, dn, count, layout, OPS[i % 3][0], inplace, R.kind_for(i, count * dt().itemsize))
    # many ownership blocks with a partial last one: 4 KiB blocks, ~100 KiB per rank
    old = L.get_param("own_block_bytes")
    R.lib.b200mpi_set_param(b"own_block_bytes", 4096)
    for algo in ("twoshot", "smem"):
        for di, dn in enumerate(("f32", "f64", "i64")):
            dt = DTYPES[dn]
            count = (n * 25 * 256 + 100) * epv(dt) + 1
            for oi, (opname, _, _) in enumerate(OPS):
                do_allreduce(R, algo, dn, count, LAYOUTS[(oi + di) % 2], opname, oi == 1, "heap")
    R.lib.b200mpi_set_param(b"own_block_bytes", old)
    R.lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)


def do_reduce(R, dn, count, layout, opname, root, inplace, kind, algo="twoshot", used=L.ALGO_TWOSHOT):
    lib, rank, n = R.lib, R.rank, R.n
    dt = DTYPES[dn]
    op, oop = {o[0]: (o[1], o[2]) for o in OPS}[opname]
    call = R.next_call("reduce")
    offs = layout_offsets(layout, dt, n, call)
    if inplace:
        offs = [(s, s) for s, _ in offs]
    ins = gen_values(dt, n, count, call)
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS[algo])
    send = Guarded(kind, dt, count, offs[rank][0], rank, call, body=ins[rank])
    recv = send if inplace else Guarded(kind, dt, count, offs[rank][1], rank, call + 1)
    mpi.Reduce(send.view, recv.view, op, root)
    order = O.ORDER_F64 if used == L.ALGO_NVLS and opname == "sum" and dn != "i64" else O.ORDER_RANK
    what = R.what("reduce", used, dt, opname, count, layout, offs, kind, inplace, root)
    if rank == root:
        recv.set_body(O.allreduce(ins, op=oop, order=order))
        check(recv, what + " [root recv]", mode_for(opname, dt, order), ins)
    else:
        check(recv, what + " [non-root recv must not be written]")
    if not inplace:
        check(send, what + " [send must be unchanged]")
        recv.free()
    send.free()


def part_reduce(R):
    n = R.n
    for di, dn in enumerate(("f32", "f64", "i64")):
        dt = DTYPES[dn]
        for ci, count in enumerate(counts_for(dt, allreduce_passes("twoshot", n, dt), R.trim)):
            for li, layout in enumerate(LAYOUTS):
                i = ci + li + di
                # small counts: over dtypes x layouts every root comes up; larger ones alternate 0 and n-1
                root = (di * len(LAYOUTS) + li + ci) % n if count <= 4097 else (0, n - 1)[i % 2]
                inplace = layout in ("aligned", "mixed") and ci % 2 == 1
                do_reduce(R, dn, count, layout, OPS[i % 3][0], root, inplace, R.kind_for(i, count * dt().itemsize))
    R.lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)


def do_reduce_scatter(R, dn, count, layout, opname, inplace, kind, algo="twoshot"):
    lib, rank, n = R.lib, R.rank, R.n
    dt = DTYPES[dn]
    op, oop = {o[0]: (o[1], o[2]) for o in OPS}[opname]
    call = R.next_call("reduce_scatter")
    offs = layout_offsets(layout, dt, n, call)
    if inplace:
        offs = [(s, s + rank * count * np.dtype(dt).itemsize) for s, _ in offs]
    ins = gen_values(dt, n, count * n, call)
    lib.b200mpi_set_algo(L.COLL_REDUCE_SCATTER, ALGOS[algo])
    used = lib.b200mpi_get_algo(L.COLL_REDUCE_SCATTER, count, O.NP2DT[np.dtype(dt)]) if opname == "sum" else L.ALGO_TWOSHOT
    order = O.ORDER_F64 if used == L.ALGO_NVLS and dn != "i64" else O.ORDER_RANK
    want = O.reduce_scatter(ins, rank, op=oop, order=order)
    send = Guarded(kind, dt, count * n, offs[rank][0], rank, call, body=ins[rank])
    what = R.what("reduce_scatter", used, dt, opname, count, layout, offs, kind, inplace)
    blocks = [x[rank * count:(rank + 1) * count] for x in ins]
    if inplace:
        mpi.ReduceScatter(send.view, send.sub(rank * count, (rank + 1) * count), op)
        send.set_body(want, rank * count)
        check(send, what + " [send with its own block reduced]", mode_for(opname, dt, order), blocks, lo=rank * count)
    else:
        recv = Guarded(kind, dt, count, offs[rank][1], rank, call + 1)
        mpi.ReduceScatter(send.view, recv.view, op)
        recv.set_body(want)
        check(recv, what + " [recv]", mode_for(opname, dt, order), blocks)
        check(send, what + " [send must be unchanged]")
        recv.free()
    send.free()


def part_reduce_scatter(R):
    for di, dn in enumerate(("f32", "f64", "i64")):
        dt = DTYPES[dn]
        for ci, count in enumerate(counts_for(dt, [1024], R.trim)):  # grid_for(count / EPV, 2)
            for li, layout in enumerate(LAYOUTS):
                i = ci + li + di
                inplace = layout in ("aligned", "mixed") and ci % 2 == 1
                do_reduce_scatter(R, dn, count, layout, OPS[i % 3][0], inplace, R.kind_for(i, count * R.n * dt().itemsize))
    R.lib.b200mpi_set_algo(L.COLL_REDUCE_SCATTER, 0)


def do_bcast(R, algo, dn, count, layout, root, kind, nvls2=None):
    lib, rank, n = R.lib, R.rank, R.n
    dt = DTYPES[dn]
    call = R.next_call("bcast")
    offs = layout_offsets(layout, dt, n, call)
    ins = gen_values(dt, n, count, call)
    if nvls2 is not None:
        lib.b200mpi_set_param(b"bcast_nvls2", nvls2)
    lib.b200mpi_set_algo(L.COLL_BCAST, ALGOS[algo])
    used = lib.b200mpi_get_algo(L.COLL_BCAST, count, O.NP2DT[np.dtype(dt)])
    buf = Guarded(kind, dt, count, offs[rank][0], rank, call, body=ins[root] if rank == root else None)
    mpi.Bcast(buf.view, root)
    buf.set_body(ins[root])
    what = R.what("bcast" if nvls2 is None else "bcast(nvls2=%d)" % nvls2, used, dt, "-", count, layout, [s for s, _ in offs], kind, True, root)
    check(buf, what)
    buf.free()


def do_allgather(R, algo, dn, count, layout, inplace, kind):
    lib, rank, n = R.lib, R.rank, R.n
    dt = DTYPES[dn]
    call = R.next_call("allgather")
    offs = layout_offsets(layout, dt, n, call)
    if inplace:
        offs = [(r_ + rank * count * np.dtype(dt).itemsize, r_) for _, r_ in offs]
    ins = gen_values(dt, n, count, call)
    lib.b200mpi_set_algo(L.COLL_ALLGATHER, ALGOS[algo])
    used = lib.b200mpi_get_algo(L.COLL_ALLGATHER, count, O.NP2DT[np.dtype(dt)])
    recv = Guarded(kind, dt, count * n, offs[rank][1], rank, call + 1)
    what = R.what("allgather", used, dt, "-", count, layout, offs, kind, inplace)
    if inplace:
        recv.set_body(ins[rank], rank * count)
        recv.load()
        mpi.Allgather(recv.sub(rank * count, (rank + 1) * count), recv.view)
    else:
        send = Guarded(kind, dt, count, offs[rank][0], rank, call, body=ins[rank])
        mpi.Allgather(send.view, recv.view)
        check(send, what + " [send must be unchanged]")
        send.free()
    recv.set_body(O.allgather(ins))
    check(recv, what + " [recv]")
    recv.free()


def do_alltoall(R, dn, count, layout, kind):
    rank, n = R.rank, R.n
    dt = DTYPES[dn]
    call = R.next_call("alltoall")
    offs = layout_offsets(layout, dt, n, call)
    ins = gen_values(dt, n, count * n, call)
    send = Guarded(kind, dt, count * n, offs[rank][0], rank, call, body=ins[rank])
    recv = Guarded(kind, dt, count * n, offs[rank][1], rank, call + 1)
    mpi.Alltoall(send.view, recv.view)
    what = R.what("alltoall", 0, dt, "-", count, layout, offs, kind)
    recv.set_body(O.alltoall(ins, rank))
    check(recv, what + " [recv]")
    check(send, what + " [send must be unchanged]")
    send.free()
    recv.free()


def part_bytes(R):
    """Bcast (both P2P modes), Allgather (push and ring) and Alltoall over u8, f32 and i64."""
    n = R.n
    for di, dn in enumerate(("u8", "f32", "i64")):
        dt = DTYPES[dn]
        es = dt().itemsize
        # grids of bytes/16 + 1 and nvec/(n-1) + 1 units, 2048 units per CTA
        for algo, passes in (("oneshot", [2047]), ("twoshot", [2047 * (n - 1)])):
            for ci, count in enumerate(counts_for(dt, passes, R.trim)):
                for li, layout in enumerate(LAYOUTS):
                    i = ci + li + di
                    do_bcast(R, algo, dn, count, layout, (i + n // 2) % n, R.kind_for(i, count * es))
        R.lib.b200mpi_set_algo(L.COLL_BCAST, 0)
        for algo in ("oneshot", "ring"):
            for ci, count in enumerate(counts_for(dt, [2047], R.trim)):
                for li, layout in enumerate(LAYOUTS):
                    i = ci + li + di
                    do_allgather(R, algo, dn, count, layout, layout in ("aligned", "mixed") and ci % 2 == 1, R.kind_for(i, count * n * es))
        R.lib.b200mpi_set_algo(L.COLL_ALLGATHER, 0)
        for ci, count in enumerate(counts_for(dt, [2047], R.trim)):
            for li, layout in enumerate(LAYOUTS):
                do_alltoall(R, dn, count, layout, R.kind_for(ci + li + di, count * n * es))


def part_v(R, counts=None, skew=None):
    """Gatherv and Scatterv (through the C ABI, so that every rank passes both buffers), Allgatherv and
    Alltoallv on skewed tables (counts and skew, when given, replace the default tables)."""
    lib, rank, n = R.lib, R.rank, R.n
    given = counts is not None
    counts = counts if given else v_tables(n)[4]  # one rank carries 70001 elements, the others 5 + r
    skew = skew if skew is not None else dict(AV.tables(n, SEED))["one pair"]
    if R.trim == "edges" and not given:
        counts = [c if c < 1000 else 4099 for c in counts]
        skew = [[c if c < 1000 else 4099 for c in row] for row in skew]
    total = sum(counts)
    displ = np.concatenate([[0], np.cumsum(counts)]).astype(int)
    tab = (ctypes.c_size_t * n)(*counts)
    for di, dn in enumerate(("u8", "f32", "i64")):
        dt = DTYPES[dn]
        for li, layout in enumerate(LAYOUTS):
            kind = "host" if (li + di) % 4 == 3 else "heap"
            mk = L.HOST if kind == "host" else L.DEVICE
            for root in sorted({0, n - 1}):
                # Gatherv: only root's recv is written
                call = R.next_call("gatherv")
                offs = layout_offsets(layout, dt, n, call)
                ins = [x[:counts[r]] for r, x in enumerate(gen_values(dt, n, max(counts), call))]
                send = Guarded(kind, dt, counts[rank], offs[rank][0], rank, call, body=ins[rank])
                recv = Guarded(kind, dt, total, offs[rank][1], rank, call + 1)
                rc = lib.b200mpi_gatherv(send.ptr(), recv.ptr(), tab, O.NP2DT[np.dtype(dt)], root, mk)
                what = R.what("gatherv", 0, dt, "-", total, layout, offs, kind, root=root) + " counts=%s" % counts
                if rc:
                    raise AssertionError("%s: %s" % (what, L.last_error()))
                if rank == root:
                    recv.set_body(G.gatherv(ins))
                check(recv, what + (" [root recv]" if rank == root else " [non-root recv must not be written]"))
                check(send, what + " [send must be unchanged]")
                send.free()
                recv.free()
                # Scatterv: root's send is read only, every recv gets its block
                call = R.next_call("scatterv")
                offs = layout_offsets(layout, dt, n, call)
                whole = gen_values(dt, 1, total, call)[0]
                send = Guarded(kind, dt, total, offs[rank][0], rank, call, body=whole if rank == root else None)
                recv = Guarded(kind, dt, counts[rank], offs[rank][1], rank, call + 1)
                rc = lib.b200mpi_scatterv(send.ptr(), recv.ptr(), tab, O.NP2DT[np.dtype(dt)], root, mk)
                what = R.what("scatterv", 0, dt, "-", total, layout, offs, kind, root=root) + " counts=%s" % counts
                if rc:
                    raise AssertionError("%s: %s" % (what, L.last_error()))
                recv.set_body(G.scatterv(whole, counts, rank))
                check(recv, what + " [recv]")
                check(send, what + (" [root send must be unchanged]" if rank == root else " [non-root send must not be written]"))
                send.free()
                recv.free()
            # Allgatherv
            call = R.next_call("allgatherv")
            offs = layout_offsets(layout, dt, n, call)
            ins = [x[:counts[r]] for r, x in enumerate(gen_values(dt, n, max(counts), call))]
            send = Guarded(kind, dt, counts[rank], offs[rank][0], rank, call, body=ins[rank])
            recv = Guarded(kind, dt, total, offs[rank][1], rank, call + 1)
            mpi.Allgatherv(send.view, recv.view, counts)
            what = R.what("allgatherv", 0, dt, "-", total, layout, offs, kind) + " counts=%s" % counts
            recv.set_body(G.gatherv(ins))
            check(recv, what + " [recv]")
            check(send, what + " [send must be unchanged]")
            send.free()
            recv.free()
            # Alltoallv
            call = R.next_call("alltoallv")
            offs = layout_offsets(layout, dt, n, call)
            row, col = AV.row(skew, rank), AV.col(skew, rank)
            sends = [gen_values(dt, 1, sum(AV.row(skew, r)), call * 8 + r)[0] for r in range(n)]
            send = Guarded(kind, dt, sum(row), offs[rank][0], rank, call, body=sends[rank])
            recv = Guarded(kind, dt, sum(col), offs[rank][1], rank, call + 1)
            mpi.Alltoallv(send.view, row, recv.view, col)
            what = R.what("alltoallv", 0, dt, "-", sum(col), layout, offs, kind) + " table=one pair"
            recv.set_body(AV.alltoallv(sends, skew, rank))
            check(recv, what + " [recv]")
            check(send, what + " [send must be unchanged]")
            send.free()
            recv.free()


def part_p2p(R):
    """Send / Receive between ranks 2k and 2k+1 into a heap sub-slice and into a host view at odd
    offsets, with room for 3 more elements than arrive: the extra room must stay unwritten."""
    rank, n = R.rank, R.n
    if rank >= n - n % 2:
        return
    peer = rank ^ 1
    for dn, offs in (("u8", (1, 7, 13)), ("f32", (4, 12, 4))):
        dt = DTYPES[dn]
        for kind in ("heap", "host"):
            for count, off in zip((1, 1001, 70001), offs):
                call = R.next_call("p2p")
                x = gen_values(dt, 1, count, call * 2 + (rank & ~1))[0]
                what = "send/receive %s count=%d kind=%s offset=%d ranks %d->%d" % (dn, count, kind, off, rank & ~1, (rank & ~1) + 1)
                if rank % 2 == 0:
                    send = Guarded(kind, dt, count, off, rank, call, body=x)
                    mpi.Send(send.view, peer, 40)
                    check(send, what + " [send must be unchanged]")
                    send.free()
                else:
                    recv = Guarded(kind, dt, count + 3, off, rank, call)
                    got = mpi.Receive(recv.view, peer, 40)
                    if len(got) != count:
                        raise AssertionError("%s: received %d elements" % (what, len(got)))
                    recv.set_body(x)
                    check(recv, what + " [recv: message, then 3 elements that must not be written]")
                    recv.free()


def part_nvls(R):
    """The switch paths: NVLS and hybrid Allreduce (i64 MAX / MIN included), the NVLS Reduce with
    asymmetric offsets (its two-shot fallback), ReduceScatter and both NVLS Bcasts."""
    lib, n = R.lib, R.n
    if not R.nvls:
        R.skipped.update(["allreduce:nvls", "allreduce:hybrid", "reduce:nvls", "reduce_scatter:nvls", "bcast:nvls", "bcast:nvls_root"])
        return
    saved = {k: L.get_param(k) for k in ("hybrid_p2p_permille", "hybrid_min_bytes", "nvls_min_ranks", "bcast_nvls2")}
    lib.b200mpi_set_param(b"hybrid_p2p_permille", 250)
    lib.b200mpi_set_param(b"hybrid_min_bytes", 0)
    lib.b200mpi_set_param(b"nvls_min_ranks", 2)
    cases = [("f32", "sum"), ("f64", "sum"), ("i64", "sum"), ("i64", "max"), ("i64", "min")]
    for algo in ("nvls", "hybrid"):
        for dn, opname in cases:
            for ci, count in enumerate((1, 257, 4097, 40001, 1048577)):
                layout = LAYOUTS[ci % 3]
                do_allreduce(R, algo, dn, count, layout, opname, ci % 2 == 1, "heap")
    for dn, opname in cases:
        for ci, count in enumerate((5, 4097, 40001)):
            for layout in ("aligned", "mixed", "split"):
                root = (ci + len(layout)) % n
                do_reduce(R, dn, count, layout, opname, root, False, "heap", algo="auto", used=L.ALGO_NVLS)
    for dn in ("f32", "i64"):
        for ci, count in enumerate((1, 4099, 262144)):
            do_reduce_scatter(R, dn, count, LAYOUTS[ci % 3], "sum", ci == 1, "heap", algo="nvls")
    for nvls2 in (0, 1):
        for dn in ("u8", "f32"):
            for ci, count in enumerate((16, 4096, 65536 * 4 + 16)):
                do_bcast(R, "nvls", dn, count, LAYOUTS[ci % 2], (ci + nvls2) % n, "heap", nvls2=nvls2)
    for k, v in saved.items():
        lib.b200mpi_set_param(k.encode(), v)
    for coll in (L.COLL_ALLREDUCE, L.COLL_BCAST, L.COLL_REDUCE_SCATTER):
        lib.b200mpi_set_algo(coll, 0)


PARTS = {"allreduce": part_allreduce, "reduce": part_reduce, "reduce_scatter": part_reduce_scatter,
         "bytes": part_bytes, "v": part_v, "p2p": part_p2p, "nvls": part_nvls}


def parse_options(argv):
    """--parts (comma list of PARTS) and --trim (counts_for) -> (options, the other arguments)."""
    ap = argparse.ArgumentParser(add_help=False)
    ap.add_argument("--parts", default=",".join(PARTS))
    ap.add_argument("--trim", default="full", choices=("full", "lean", "edges"), help="counts per kernel (counts_for)")
    return ap.parse_known_args(argv)


def scenario_footprint(a, opts=None):
    """opts: parse_options' result; every part at full counts when omitted."""
    opts = opts if opts is not None else parse_options([])[0]
    R = Run(opts)
    secs = {}
    for name in opts.parts.split(","):
        t0 = time.time()
        PARTS[name](R)
        mpi.Barrier()
        secs[name] = round(time.time() - t0, 2)
    return {"checked": R.call, "by_part": R.done, "seconds": secs, "nvls": R.nvls, "skipped": sorted(R.skipped)}


W.SCENARIOS.update({k[len("scenario_"):]: v for k, v in list(globals().items()) if k.startswith("scenario_")})

if __name__ == "__main__":
    opts, rest = parse_options(sys.argv[1:])
    sys.argv = [sys.argv[0]] + rest  # _worker.main parses the rest
    W.SCENARIOS["footprint"] = lambda a: scenario_footprint(a, opts)
    W.main()
