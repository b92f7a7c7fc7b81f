"""One rank of a test world in which the ranks of one call pass different kinds of buffer.
Usage as _worker.py: _kinds_worker.py kinds --out FILE [--parts ...] [--trim full|lean] -mpi-* flags.

The kind of rank r on call i is KINDS[(r + i) % len(KINDS)]: heap views (mpi.Alloc) and torch CUDA
tensors wrapped as DeviceSlice(owner=False), each at a 16-byte-aligned and a misaligned offset; a heap
send with a torch recv and the reverse; pinned host memory from b200mpi_host_alloc and from a torch
pin_memory tensor; pageable numpy.  Device ranks and host ranks of one call stage differently but must
launch the same kernels, so every rank checks every buffer it passed, guards included, bit for bit
against the oracle in the order of the kernel that ran.  Part 'hostpipe' runs the chunked host-slice
pipeline with pageable, pinned and registered ranks in one call (see pipe_calls)."""
import argparse
import ctypes
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _alltoallv_ref as AV  # noqa: E402
import _footprint_worker as F  # noqa: E402
import _gather_oracle as G  # noqa: E402
import _worker as W  # noqa: E402
from _rsv_ref import rsv_oracle  # noqa: E402
from _scan_ref import scan_oracle  # noqa: E402
from _worker import ALGOS, L, O, SEED, expect_allreduce, mpi  # noqa: E402

DTYPES = F.DTYPES
OPS = {name: (op, oop) for name, op, oop in F.OPS}
OPNAMES = [o[0] for o in F.OPS]
DEVICE_STORAGE = ("heap", "torch")
# (send storage, recv storage, misaligned)
KINDS = (("heap", "heap", False), ("heap", "heap", True), ("torch", "torch", False), ("torch", "torch", True),
         ("heap", "torch", False), ("torch", "heap", True), ("pinned", "pinned", False), ("torchpin", "torchpin", True),
         ("pageable", "pageable", False))
MISALIGN = {1: 7, 4: 4, 8: 8}  # byte offset of a misaligned view: element-aligned, not 16-byte aligned

# The pipelined host-slice part: knobs under which the pipe and bounce chunks differ, the memory each
# rank passes (rotated per call), and which ranks pin pageable memory in place or run no copy threads.
PIPE_KNOBS = (("pipe_min_bytes", 64 << 10), ("pipe_chunk_bytes", 1 << 20), ("bounce_chunk_bytes", 256 << 10))
PIPE_MEMS = ("pageable", "pinned", "torchpin")
PIPE_CASES = (("f32", 300001), ("i64", 150001))


def pipe_env(n, r):
    """Rank 1 registers pageable buffers (cudaHostRegister); in worlds of 3 and more rank n-1 has no
    copy threads, so its pageable buffers take the direct DMA path."""
    e = {}
    if r == 1:
        e["B200MPI_HOST_REGISTER"] = "1"
    if n >= 3 and r == n - 1:
        e["B200MPI_HOST_THREADS"] = "0"
    return e


def pipe_bounces(n, r, mem):
    """Whether rank r's buffer of kind `mem` goes through the bounce ring (pageable, not registered,
    copy threads running)."""
    return mem == "pageable" and not pipe_env(n, r)


def pipe_calls(n, cases=PIPE_CASES):
    """[(call index, collective, dtype name, count, rows, extra)] of part hostpipe, in order; rank r
    passes PIPE_MEMS[(r + call index) % 3] on each."""
    out = []
    for dn, count in cases:
        for coll, extra in (("allreduce", "twoshot"), ("allreduce", "twoshot inplace"), ("bcast", 0), ("bcast", n - 1),
                            ("allgather", None), ("allreduce", "auto")):
            out.append((len(out), coll, dn, count, n if coll == "allgather" else 1, extra))
    return out


def torch_mod():
    import torch
    torch.cuda.set_device(L.load().b200mpi_device())
    return torch


class Buf(F.Guarded):
    """F.Guarded over any storage: `count` elements at byte `off` past the head guard."""

    def __init__(self, storage, dt, count, off, rank, call, body=None):
        self.storage, self.dt, self.count, self.off = storage, np.dtype(dt), int(count), int(off)
        self.kind = "heap" if storage in DEVICE_STORAGE else "host"
        self.head, self.nbody, self.tail, self.total = F.zones(count, dt, off)
        self.image = F.guard_pattern(rank, call, self.total)
        if body is not None:
            self.set_body(body)
        self.hp = None
        if storage == "heap":
            self.mem = mpi.Alloc(self.total, np.uint8)
            base = self.mem.ptr
        elif storage == "torch":
            torch = torch_mod()
            self.mem = torch.empty(self.total, dtype=torch.uint8, device="cuda")
            base = self.mem.data_ptr()
        elif storage == "pinned":
            self.mem, self.hp = W.pinned_array(self.total, np.uint8)
        elif storage == "torchpin":
            torch = torch_mod()
            self.pin = torch.empty(self.total, dtype=torch.uint8, pin_memory=True)
            self.mem = self.pin.numpy()
        else:
            raw = np.empty(self.total + 64, dtype=np.uint8)
            s = (-raw.ctypes.data) % 64
            self.mem = raw[s:s + self.total]
        self.load()
        if self.kind == "heap":
            self.view = mpi.DeviceSlice(self.count, self.dt, base + self.head, owner=False)
        else:
            self.view = self.mem[self.head:self.head + self.nbody].view(self.dt)

    @property
    def memkind(self):
        return L.DEVICE if self.kind == "heap" else L.HOST

    def load(self):
        if self.storage == "heap":
            self.mem.copy_from_host(self.image)
        elif self.storage == "torch":
            torch = torch_mod()
            self.mem.copy_(torch.from_numpy(self.image))
            torch.cuda.synchronize()
        else:
            self.mem[:] = self.image

    def read(self):
        if self.storage == "heap":
            return self.mem.to_host()
        if self.storage == "torch":
            torch_mod().cuda.synchronize()
            return self.mem.cpu().numpy()
        return np.array(self.mem, copy=True)

    def free(self):
        if self.storage == "heap":
            self.mem.free()
        elif self.hp is not None:
            L.load().b200mpi_host_free(self.hp)
            self.hp = None
        self.mem = self.view = None


class Inner:
    """`count` elements `lo` elements into a Buf: the inner buffer of an in-place call."""

    def __init__(self, outer, lo, count):
        self.view, self.memkind = outer.sub(lo, lo + count), outer.memkind

    def ptr(self):
        if isinstance(self.view, mpi.DeviceSlice):
            return self.view.ptr
        return self.view.ctypes.data if self.view.size else None


class Run:
    def __init__(self, a):
        self.lib = L.load()
        self.rank, self.n = mpi.Rank(), mpi.Size()
        self.call = 0
        self.done = {}
        self.trim = a.trim

    def next_call(self, part):
        self.call += 1
        self.done[part] = self.done.get(part, 0) + 1
        return self.call

    def kinds(self, call, r=None):
        return KINDS[((self.rank if r is None else r) + call) % len(KINDS)]

    def offsets(self, call, dt):
        """(send, recv) byte offsets of this rank on `call`: 0 or MISALIGN, plus 16 on odd ranks."""
        mis = self.kinds(call)[2]
        o = (MISALIGN[np.dtype(dt).itemsize] if mis else 0) + 16 * (self.rank % 2)
        return o, o

    def buf(self, call, dt, count, body=None):
        """One buffer of this rank's send storage (Bcast)."""
        return Buf(self.kinds(call)[0], dt, count, self.offsets(call, dt)[0], self.rank, call, body=body)

    def bufs(self, call, dt, scount, rcount, body=None, inplace_at=None):
        """(send, recv) of this rank.  inplace_at: None, two buffers; "same", one buffer for both; an
        int >= 0, send is the Inner view that many elements into recv (filled with body); an int < 0,
        recv is the Inner view -inplace_at - 1 elements into send."""
        ss, rs, _ = self.kinds(call)
        so, ro = self.offsets(call, dt)
        if inplace_at is None:
            return Buf(ss, dt, scount, so, self.rank, call, body=body), Buf(rs, dt, rcount, ro, self.rank, call + 1)
        if inplace_at == "same":
            b = Buf(ss, dt, scount, so, self.rank, call, body=body)
            return b, b
        if inplace_at >= 0:
            outer = Buf(rs, dt, rcount, ro, self.rank, call + 1)
            if body is not None:
                outer.set_body(body, inplace_at)
                outer.load()
            return Inner(outer, inplace_at, scount), outer
        outer = Buf(ss, dt, scount, so, self.rank, call, body=body)
        return outer, Inner(outer, -inplace_at - 1, rcount)

    def what(self, coll, dt, opname, count, call, extra=""):
        ks = ["%s/%s%s" % (s, r_, "+mis" if m else "") for s, r_, m in (self.kinds(call, r) for r in range(self.n))]
        return "%s dtype=%s op=%s count=%d kinds per rank=%s rank=%d %s" % (coll, np.dtype(dt).name, opname, count, ks, self.rank, extra)


def counts_for(dt, trim):
    e = F.epv(dt)
    return [0, 1, e + 1, 4097, 65537] if trim == "full" else [1, e + 1, 4097]


def check_send(send, what):
    if isinstance(send, Buf):
        F.check(send, what + " [send must be unchanged]")


# ---- reductions ---------------------------------------------------------------------------------
def part_allreduce(R):
    lib, rank, n = R.lib, R.rank, R.n
    for ai, algo in enumerate(("oneshot", "twoshot", "smem", "ring", "ll")):
        lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS[algo])
        for di, dn in enumerate(("f32", "f64", "i64")):
            dt = DTYPES[dn]
            for ci, count in enumerate(counts_for(dt, R.trim)):
                opname = OPNAMES[(ci + di) % 3]
                op, oop = OPS[opname]
                inplace = (ai + di + ci) % 2 == 1
                call = R.next_call("allreduce")
                ins = F.gen_values(dt, n, count, call)
                used = lib.b200mpi_get_algo(L.COLL_ALLREDUCE, count, O.NP2DT[np.dtype(dt)])
                send, recv = R.bufs(call, dt, count, count, body=ins[rank], inplace_at="same" if inplace else None)
                mpi.Allreduce(send.view, recv.view, op)
                want, order = expect_allreduce(ins, oop, used, n, count, dt)
                what = R.what("allreduce algo=%s" % L.ALGO_NAMES[used], dt, opname, count, call, "inplace=%s" % inplace)
                recv.set_body(want)
                F.check(recv, what + " [recv]", F.mode_for(opname, dt, order), ins)
                if not inplace:
                    check_send(send, what)
                    send.free()
                recv.free()
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)


def part_reduce(R):
    """Reduce to a non-zero root (two-shot) and ReduceScatter, in place and out of place."""
    lib, rank, n = R.lib, R.rank, R.n
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, ALGOS["twoshot"])
    for di, dn in enumerate(("f32", "f64", "i64")):
        dt = DTYPES[dn]
        for ci, count in enumerate(counts_for(dt, R.trim)):
            opname = OPNAMES[(ci + di) % 3]
            op, oop = OPS[opname]
            root = 1 + (ci + di) % (n - 1)
            inplace = (ci + di) % 2 == 1 and rank == root
            call = R.next_call("reduce")
            ins = F.gen_values(dt, n, count, call)
            send, recv = R.bufs(call, dt, count, count, body=ins[rank], inplace_at="same" if inplace else None)
            mpi.Reduce(send.view, recv.view, op, root)
            what = R.what("reduce root=%d" % root, dt, opname, count, call, "inplace=%s" % inplace)
            if rank == root:
                recv.set_body(O.allreduce(ins, op=oop, order=O.ORDER_RANK))
                F.check(recv, what + " [root recv]", F.mode_for(opname, dt, O.ORDER_RANK), ins)
            else:
                F.check(recv, what + " [non-root recv must not be written]")
            if not inplace:
                check_send(send, what)
                send.free()
            recv.free()
    lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
    for di, dn in enumerate(("f32", "f64", "i64")):
        dt = DTYPES[dn]
        for ci, count in enumerate(counts_for(dt, R.trim)):
            opname = OPNAMES[(ci + di + 1) % 3]
            op, oop = OPS[opname]
            inplace = (ci + di) % 2 == 0
            call = R.next_call("reduce_scatter")
            ins = F.gen_values(dt, n, count * n, call)
            used = lib.b200mpi_get_algo(L.COLL_REDUCE_SCATTER, count, O.NP2DT[np.dtype(dt)]) if opname == "sum" else L.ALGO_TWOSHOT
            order = O.ORDER_F64 if used == L.ALGO_NVLS and dn != "i64" else O.ORDER_RANK
            send, recv = R.bufs(call, dt, count * n, count, body=ins[rank], inplace_at=-(rank * count) - 1 if inplace else None)
            mpi.ReduceScatter(send.view, recv.view, op)
            what = R.what("reduce_scatter", dt, opname, count, call, "inplace=%s" % inplace)
            want = O.reduce_scatter(ins, rank, op=oop, order=order)
            blocks = [x[rank * count:(rank + 1) * count] for x in ins]
            if inplace:
                send.set_body(want, rank * count)
                F.check(send, what + " [send with its own block reduced]", F.mode_for(opname, dt, order), blocks, lo=rank * count)
            else:
                recv.set_body(want)
                F.check(recv, what + " [recv]", F.mode_for(opname, dt, order), blocks)
                check_send(send, what)
                recv.free()
            send.free()


def part_scan(R):
    """Scan and Exscan, in place and out of place; rank 0's Exscan recv must not be written."""
    rank, n = R.rank, R.n
    for exclusive in (False, True):
        for di, dn in enumerate(("f32", "f64", "i64")):
            dt = DTYPES[dn]
            for ci, count in enumerate(counts_for(dt, R.trim)):
                opname = OPNAMES[(ci + di + exclusive) % 3]
                op, oop = OPS[opname]
                inplace = (ci + di) % 2 == 1
                call = R.next_call("exscan" if exclusive else "scan")
                ins = F.gen_values(dt, n, count, call)
                send, recv = R.bufs(call, dt, count, count, body=ins[rank], inplace_at="same" if inplace else None)
                (mpi.Exscan if exclusive else mpi.Scan)(send.view, recv.view, op)
                what = R.what("exscan" if exclusive else "scan", dt, opname, count, call, "inplace=%s" % inplace)
                want = scan_oracle(ins, oop, rank, exclusive)
                if want is None:  # rank 0 of an Exscan: in place it keeps its input
                    F.check(recv, what + " [rank 0 recv must not be written]")
                else:
                    recv.set_body(want)
                    F.check(recv, what + " [recv]", F.mode_for(opname, dt, O.ORDER_RANK), ins[:rank + (0 if exclusive else 1)])
                if not inplace:
                    check_send(send, what)
                    send.free()
                recv.free()


def part_rsv(R):
    """ReduceScatterv over tables that put every count on every rank; a rank whose block is 0 passes a
    NULL recv, and its send must come back unchanged."""
    lib, rank, n = R.lib, R.rank, R.n
    for di, dn in enumerate(("f32", "f64", "i64")):
        dt = DTYPES[dn]
        cs = counts_for(dt, R.trim)
        for ci in range(len(cs)):
            counts = [cs[(r + ci) % len(cs)] for r in range(n)]
            d = [int(x) for x in np.concatenate([[0], np.cumsum(counts)])]
            opname = OPNAMES[(ci + di) % 3]
            op, oop = OPS[opname]
            inplace = (ci + di) % 2 == 1 and counts[rank] > 0
            call = R.next_call("reduce_scatterv")
            ins = F.gen_values(dt, n, d[-1], call)
            send, recv = R.bufs(call, dt, d[-1], counts[rank], body=ins[rank], inplace_at=-d[rank] - 1 if inplace else None)
            null = counts[rank] == 0 and (ci + di) % 2 == 0
            tab = (ctypes.c_size_t * n)(*counts)
            rc = lib.b200mpi_reduce_scatterv(send.ptr(), None if null else recv.ptr(), tab, O.NP2DT[np.dtype(dt)], op, send.memkind)
            what = R.what("reduce_scatterv counts=%s" % counts, dt, opname, d[-1], call, "inplace=%s null_recv=%s" % (inplace, null))
            if rc:
                raise AssertionError("%s: %s" % (what, L.last_error()))
            want = rsv_oracle(ins, counts, oop, rank)
            blocks = [x[d[rank]:d[rank + 1]] for x in ins]
            if inplace:
                send.set_body(want, d[rank])
                F.check(send, what + " [send with its own block reduced]", F.mode_for(opname, dt, O.ORDER_RANK), blocks, lo=d[rank])
            else:
                recv.set_body(want)
                F.check(recv, what + (" [recv must not be written]" if null else " [recv]"), F.mode_for(opname, dt, O.ORDER_RANK), blocks)
                check_send(send, what)
                recv.free()
            send.free()


# ---- byte movers --------------------------------------------------------------------------------
def part_bytes(R):
    """Both P2P Bcasts, push and ring Allgather, Alltoall over u8, f32 and i64."""
    lib, rank, n = R.lib, R.rank, R.n
    for di, dn in enumerate(("u8", "f32", "i64")):
        dt = DTYPES[dn]
        for ai, algo in enumerate(("oneshot", "twoshot")):
            lib.b200mpi_set_algo(L.COLL_BCAST, ALGOS[algo])
            for ci, count in enumerate(counts_for(dt, R.trim)):
                root = (ci + ai + di) % n
                call = R.next_call("bcast")
                x = F.gen_values(dt, 1, count, call)[0]
                buf = R.buf(call, dt, count, body=x if rank == root else None)
                mpi.Bcast(buf.view, root)
                buf.set_body(x)
                F.check(buf, R.what("bcast algo=%s root=%d" % (algo, root), dt, "-", count, call))
                buf.free()
        lib.b200mpi_set_algo(L.COLL_BCAST, 0)
        for ai, algo in enumerate(("oneshot", "ring")):
            lib.b200mpi_set_algo(L.COLL_ALLGATHER, ALGOS[algo])
            for ci, count in enumerate(counts_for(dt, R.trim)):
                inplace = (ci + ai + di) % 2 == 1
                call = R.next_call("allgather")
                ins = F.gen_values(dt, n, count, call)
                send, recv = R.bufs(call, dt, count, count * n, body=ins[rank], inplace_at=rank * count if inplace else None)
                mpi.Allgather(send.view, recv.view)
                what = R.what("allgather algo=%s" % algo, dt, "-", count, call, "inplace=%s" % inplace)
                recv.set_body(O.allgather(ins))
                F.check(recv, what + " [recv]")
                if not inplace:
                    check_send(send, what)
                    send.free()
                recv.free()
        lib.b200mpi_set_algo(L.COLL_ALLGATHER, 0)
        for ci, count in enumerate(counts_for(dt, R.trim)):
            call = R.next_call("alltoall")
            ins = F.gen_values(dt, n, count * n, call)
            send, recv = R.bufs(call, dt, count * n, count * n, body=ins[rank])
            mpi.Alltoall(send.view, recv.view)
            what = R.what("alltoall", dt, "-", count, call)
            recv.set_body(O.alltoall(ins, rank))
            F.check(recv, what + " [recv]")
            check_send(send, what)
            send.free()
            recv.free()


def part_rooted(R):
    """Gather, Scatter, Gatherv, Scatterv (every rank passes both buffers through the C ABI, so the one
    a rank does not use is checked unchanged), Allgatherv, and Alltoallv on a skewed table."""
    lib, rank, n = R.lib, R.rank, R.n
    skew = dict(AV.tables(n, SEED))["one pair"]
    for di, dn in enumerate(("u8", "f32", "i64")):
        dt = DTYPES[dn]
        code = O.NP2DT[np.dtype(dt)]
        cs = counts_for(dt, R.trim)
        for ci, c in enumerate(cs):
            root = (ci + di) % n
            inplace = (ci + di) % 2 == 1 and rank == root
            counts = [cs[(r + ci) % len(cs)] for r in range(n)]
            d = [int(x) for x in np.concatenate([[0], np.cumsum(counts)])]
            tab = (ctypes.c_size_t * n)(*counts)
            for coll in ("gather", "gatherv"):
                v = coll == "gatherv"
                mine, total = (counts[rank], d[-1]) if v else (c, c * n)
                at = d[rank] if v else rank * c
                call = R.next_call(coll)
                ins = [x[:(counts[r] if v else c)] for r, x in enumerate(F.gen_values(dt, n, max(counts) if v else c, call))]
                send, recv = R.bufs(call, dt, mine, total, body=ins[rank], inplace_at=at if inplace else None)
                rc = (lib.b200mpi_gatherv(send.ptr(), recv.ptr(), tab, code, root, recv.memkind) if v else
                      lib.b200mpi_gather(send.ptr(), recv.ptr(), c, code, root, recv.memkind))
                what = R.what("%s root=%d" % (coll, root) + (" counts=%s" % counts if v else ""), dt, "-", total, call, "inplace=%s" % inplace)
                if rc:
                    raise AssertionError("%s: %s" % (what, L.last_error()))
                if rank == root:
                    recv.set_body(G.gatherv(ins))
                F.check(recv, what + (" [root recv]" if rank == root else " [non-root recv must not be written]"))
                if not inplace:
                    check_send(send, what)
                    send.free()
                recv.free()
            for coll in ("scatter", "scatterv"):
                v = coll == "scatterv"
                tcounts = counts if v else [c] * n
                td = [int(x) for x in np.concatenate([[0], np.cumsum(tcounts)])]
                call = R.next_call(coll)
                whole = F.gen_values(dt, 1, td[-1], call)[0]
                send, recv = R.bufs(call, dt, td[-1], tcounts[rank], body=whole if rank == root else None,
                                    inplace_at=-td[rank] - 1 if inplace else None)
                rc = (lib.b200mpi_scatterv(send.ptr(), recv.ptr(), tab, code, root, send.memkind) if v else
                      lib.b200mpi_scatter(send.ptr(), recv.ptr(), c, code, root, send.memkind))
                what = R.what("%s root=%d" % (coll, root) + (" counts=%s" % counts if v else ""), dt, "-", td[-1], call, "inplace=%s" % inplace)
                if rc:
                    raise AssertionError("%s: %s" % (what, L.last_error()))
                if inplace:
                    F.check(send, what + " [root send, its own block in place]")
                else:
                    recv.set_body(G.scatterv(whole, tcounts, rank))
                    F.check(recv, what + " [recv]")
                    F.check(send, what + (" [root send must be unchanged]" if rank == root else " [non-root send must not be written]"))
                    recv.free()
                send.free()
            # Allgatherv
            inplace = (ci + di) % 2 == 0
            call = R.next_call("allgatherv")
            ins = [x[:counts[r]] for r, x in enumerate(F.gen_values(dt, n, max(counts), call))]
            send, recv = R.bufs(call, dt, counts[rank], d[-1], body=ins[rank], inplace_at=d[rank] if inplace else None)
            mpi.Allgatherv(send.view, recv.view, counts)
            what = R.what("allgatherv counts=%s" % counts, dt, "-", d[-1], call, "inplace=%s" % inplace)
            recv.set_body(G.gatherv(ins))
            F.check(recv, what + " [recv]")
            if not inplace:
                check_send(send, what)
                send.free()
            recv.free()
        # Alltoallv on the skewed table
        call = R.next_call("alltoallv")
        row, col = AV.row(skew, rank), AV.col(skew, rank)
        sends = [F.gen_values(dt, 1, sum(AV.row(skew, r)), call * 8 + r)[0] for r in range(n)]
        send, recv = R.bufs(call, dt, sum(row), sum(col), body=sends[rank])
        mpi.Alltoallv(send.view, row, recv.view, col)
        what = R.what("alltoallv table=one pair", dt, "-", sum(col), call)
        recv.set_body(AV.alltoallv(sends, skew, rank))
        F.check(recv, what + " [recv]")
        check_send(send, what)
        send.free()
        recv.free()


# ---- enqueue-only entries and mismatches on torch tensors ---------------------------------------
def part_async(R):
    """The four _async entries on torch tensors, eight calls back to back before one stream_sync, on the
    library stream and on a caller stream.  Run first in a process: within each sequence Allgather's
    recv and ReduceScatter's send outgrow the staging blocks the calls before them used, so ensure_stage
    replaces a block while the earlier calls' copy-backs are still queued.  Every tensor is filled
    before the first call: nothing synchronises the device inside a sequence."""
    torch = torch_mod()
    lib, rank, n = R.lib, R.rank, R.n
    base = 262145  # 1 MiB + 4 bytes of f32: above the smallest staging block
    for si, (dn, stream, count) in enumerate((("f32", False, base), ("f64", True, base), ("i64", False, 2 * base))):
        dt = DTYPES[dn]
        code = O.NP2DT[np.dtype(dt)]
        root = si % n
        calls = []  # (name, issue(send, recv), send, recv, want, mode, ins for the tolerance)

        def pair(scount, rcount, body):
            call = R.next_call(name)
            mis = MISALIGN[np.dtype(dt).itemsize] * (call % 2)
            return (Buf("torch", dt, scount, mis, rank, call, body=body) if scount is not None else None,
                    Buf("torch", dt, rcount, 16 - mis, rank, call + 1))

        for opname in OPNAMES:
            name = "allreduce_async op=%s" % opname
            ins = F.gen_values(dt, n, count, R.call + 1)
            s, r_ = pair(count, count, ins[rank])
            used = lib.b200mpi_get_algo(L.COLL_ALLREDUCE, count, code) if opname == "sum" else L.ALGO_TWOSHOT
            want, order = expect_allreduce(ins, OPS[opname][1], used, n, count, dt)
            calls.append((name, lambda s, r_, op=OPS[opname][0]: lib.b200mpi_allreduce_async(s.ptr(), r_.ptr(), count, code, op),
                          s, r_, want, F.mode_for(opname, dt, order), ins))
        name = "bcast_async root=%d" % root
        x = F.gen_values(dt, 1, count, R.call + 1)[0]
        _, b = pair(None, count, None)
        if rank == root:
            b.set_body(x)
            b.load()
        calls.append((name, lambda s, r_: lib.b200mpi_bcast_async(r_.ptr(), count, code, root), None, b, x, "exact", None))
        name = "allgather_async"
        ins = F.gen_values(dt, n, count, R.call + 1)
        s, r_ = pair(count, count * n, ins[rank])
        calls.append((name, lambda s, r_: lib.b200mpi_allgather_async(s.ptr(), r_.ptr(), count, code), s, r_, O.allgather(ins), "exact", None))
        for opname in OPNAMES:
            name = "reduce_scatter_async op=%s" % opname
            ins = F.gen_values(dt, n, count * n, R.call + 1)
            s, r_ = pair(count * n, count, ins[rank])
            used = lib.b200mpi_get_algo(L.COLL_REDUCE_SCATTER, count, code) if opname == "sum" else L.ALGO_TWOSHOT
            order = O.ORDER_F64 if used == L.ALGO_NVLS and dn != "i64" else O.ORDER_RANK
            calls.append((name, lambda s, r_, op=OPS[opname][0]: lib.b200mpi_reduce_scatter_async(s.ptr(), r_.ptr(), count, code, op),
                          s, r_, O.reduce_scatter(ins, rank, op=OPS[opname][1], order=order), F.mode_for(opname, dt, order),
                          [v[rank * count:(rank + 1) * count] for v in ins]))
        st = None
        if stream:
            st = torch.cuda.Stream()
            assert lib.b200mpi_set_stream(ctypes.c_void_p(st.cuda_stream)) == 0, L.last_error()
        what = "%s count=%d stream=%s rank=%d" % (dn, count, "caller" if stream else "library", rank)
        for name, issue, s, r_, _, _, _ in calls:
            if issue(s, r_):
                raise AssertionError("%s %s: %s" % (name, what, L.last_error()))
        rc = lib.b200mpi_stream_sync()
        if stream:
            st.synchronize()
            assert lib.b200mpi_set_stream(None) == 0
        if rc:
            raise AssertionError("stream_sync after the async sequence %s: %s" % (what, L.last_error()))
        for name, _, s, r_, want, mode, ins in calls:
            r_.set_body(want)
            F.check(r_, "%s %s [recv]" % (name, what), mode, ins)
            if s is not None:
                F.check(s, "%s %s [send must be unchanged]" % (name, what))
                s.free()
            r_.free()


def part_mismatch(R):
    """Calls on torch tensors whose counts differ between ranks get B200MPI_ERR_PEER on every rank,
    after a successful call of the same shape left its result in the staging block; the caller's
    buffers stay byte for byte as they were, and the next call works."""
    lib, rank, n = R.lib, R.rank, R.n
    old_ll = L.get_param("ll_max_bytes")
    assert lib.b200mpi_set_param(b"ll_max_bytes", 0) == 0  # the LL kernel carries no signature
    c, root = 1000, n - 1
    assert c * n * 4 < L.get_param("pipe_min_bytes")
    calls = (
        ("allreduce", c, c, lambda s, r, k: lib.b200mpi_allreduce(s, r, k, L.F32, L.SUM, L.DEVICE)),
        ("bcast", c, c, lambda s, r, k: lib.b200mpi_bcast(s if rank == 0 else r, k, L.F32, 0, L.DEVICE)),
        ("allgather", c, c * n, lambda s, r, k: lib.b200mpi_allgather(s, r, k, L.F32, L.DEVICE)),
        ("reduce_scatter", c * n, c, lambda s, r, k: lib.b200mpi_reduce_scatter(s, r, k, L.F32, L.SUM, L.DEVICE)),
        ("reduce", c, c, lambda s, r, k: lib.b200mpi_reduce(s, r, k, L.F32, L.SUM, root, L.DEVICE)),
        ("alltoall", c * n, c * n, lambda s, r, k: lib.b200mpi_alltoall(s, r, k, L.F32, L.DEVICE)),
    )
    for name, ns, nr, call_fn in calls:
        call = R.next_call("mismatch")
        send = Buf("torch", np.float32, ns, 4 * (call % 2), rank, call, body=np.arange(ns, dtype=np.float32) + 10 * (rank + 1))
        recv = Buf("torch", np.float32, nr, 4 * (call % 3 == 0), rank, call + 1)
        rc = call_fn(send.ptr(), recv.ptr(), c)
        assert rc == 0, (name, rc, L.last_error())
        recv.load()
        rc = call_fn(send.ptr(), recv.ptr(), c if rank == 0 else c - 1)
        what = "%s on torch tensors, count %d on rank %d" % (name, c if rank == 0 else c - 1, rank)
        assert rc == L.ERR_PEER, (what, rc, L.last_error())
        F.check(recv, what + " [recv must not be written by a mismatched call]")
        F.check(send, what + " [send must be unchanged]")
        send.free()
        recv.free()
    assert lib.b200mpi_set_param(b"ll_max_bytes", old_ll) == 0
    call = R.next_call("mismatch")
    ins = F.gen_values(np.float32, n, c, call)
    send, recv = Buf("torch", np.float32, c, 0, rank, call, body=ins[rank]), Buf("torch", np.float32, c, 4, rank, call + 1)
    used = lib.b200mpi_get_algo(L.COLL_ALLREDUCE, c, L.F32)
    mpi.Allreduce(send.view, recv.view, mpi.MAX)
    want, _ = expect_allreduce(ins, O.MAX, used, n, c, np.float32)
    recv.set_body(want)
    F.check(recv, "allreduce algo=%s on torch tensors after the mismatches" % L.ALGO_NAMES[used])
    send.free()
    recv.free()


# ---- pipelined host slices with mixed pinning ---------------------------------------------------
def part_hostpipe(R):
    """Allreduce (two-shot, out of place and in place, then AUTO), Bcast from the first and the last
    rank and Allgather through the chunked pipeline, while in one call some ranks pass pageable memory
    (bounced, registered or DMA'd directly, after pipe_env) and others pinned memory."""
    lib, rank, n = R.lib, R.rank, R.n
    saved = {k: L.get_param(k) for k, _ in PIPE_KNOBS + (("ll_max_bytes", 0),)}
    for k, v in PIPE_KNOBS:
        assert lib.b200mpi_set_param(k.encode(), v) == 0, L.last_error()
    keep = []  # pageable buffers stay allocated: a registered range must not be handed out again
    cases = PIPE_CASES if R.trim == "full" else PIPE_CASES[:1]
    for i, coll, dn, count, rows, extra in pipe_calls(n, cases):
        dt = DTYPES[dn]
        mem = PIPE_MEMS[(rank + i) % len(PIPE_MEMS)]
        call = R.next_call("hostpipe " + coll)
        opname = OPNAMES[i % 3]
        op, oop = OPS[opname]
        ins = F.gen_values(dt, n, count, call)
        what = "hostpipe %s %s dtype=%s op=%s count=%d mem=%s (ranks %s) rank=%d" % (
            coll, extra, dn, opname, count, mem, [PIPE_MEMS[(r + i) % len(PIPE_MEMS)] for r in range(n)], rank)
        off = 16 * (rank % 2) + (MISALIGN[np.dtype(dt).itemsize] if i % 2 else 0)
        if coll == "allreduce":
            inplace = extra == "twoshot inplace"
            auto = extra == "auto"
            lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0 if auto else ALGOS["twoshot"])
            if auto:  # the pipeline never runs the LL kernel; AUTO's answer below must not either
                lib.b200mpi_set_param(b"ll_max_bytes", 0)
                op, oop, opname = mpi.SUM, O.SUM, "sum"
            send = Buf(mem, dt, count, off, rank, call, body=ins[rank])
            recv = send if inplace else Buf(mem, dt, count, off + 16, rank, call + 1)
            mpi.Allreduce(send.view, recv.view, op)
            if auto:  # chunk by chunk: every rank chunks by the smaller knob
                ce = max(min(PIPE_KNOBS[1][1], PIPE_KNOBS[2][1]) // np.dtype(dt).itemsize, 4096) // 4096 * 4096
                want, orders = np.empty(count, dtype=dt), set()
                for lo in range(0, count, ce):
                    part = [x[lo:lo + ce] for x in ins]
                    used = lib.b200mpi_get_algo(L.COLL_ALLREDUCE, len(part[0]), O.NP2DT[np.dtype(dt)])
                    want[lo:lo + ce], o = expect_allreduce(part, O.SUM, used, n, len(part[0]), dt)
                    orders.add(o)
                mode = F.mode_for("sum", dt, O.ORDER_F64 if O.ORDER_F64 in orders else O.ORDER_RANK)
            else:
                want, mode = O.allreduce(ins, op=oop, order=O.ORDER_RANK), F.mode_for(opname, dt, O.ORDER_RANK)
            recv.set_body(want)
            F.check(recv, what + " [recv]", mode, ins)
            if not inplace:
                F.check(send, what + " [send must be unchanged]")
                keep.append(recv)
            keep.append(send)
            lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
            lib.b200mpi_set_param(b"ll_max_bytes", saved["ll_max_bytes"])
        elif coll == "bcast":
            root = extra
            buf = Buf(mem, dt, count, off, rank, call, body=ins[root] if rank == root else None)
            mpi.Bcast(buf.view, root)
            buf.set_body(ins[root])
            F.check(buf, what + " root=%d" % root)
            keep.append(buf)
        else:
            send = Buf(mem, dt, count, off, rank, call, body=ins[rank])
            recv = Buf(mem, dt, count * n, off + 16, rank, call + 1)
            mpi.Allgather(send.view, recv.view)
            recv.set_body(O.allgather(ins))
            F.check(recv, what + " [recv]")
            F.check(send, what + " [send must be unchanged]")
            keep += [send, recv]
    for k, v in saved.items():
        lib.b200mpi_set_param(k.encode(), v)
    mpi.Barrier()
    for b in keep:
        b.free()


PARTS = {"async": part_async, "allreduce": part_allreduce, "reduce": part_reduce, "scan": part_scan, "rsv": part_rsv,
         "bytes": part_bytes, "rooted": part_rooted, "mismatch": part_mismatch, "hostpipe": part_hostpipe}
DEFAULT_PARTS = "async,allreduce,reduce,scan,rsv,bytes,rooted,mismatch"


def parse_options(argv):
    ap = argparse.ArgumentParser(add_help=False)
    ap.add_argument("--parts", default=DEFAULT_PARTS)
    ap.add_argument("--trim", default="full", choices=("full", "lean"), help="counts per call (counts_for)")
    return ap.parse_known_args(argv)


def scenario_kinds(a, opts=None):
    opts = opts if opts is not None else parse_options([])[0]
    R = Run(opts)
    secs = {}
    for name in opts.parts.split(","):
        t0 = time.time()
        PARTS[name](R)
        mpi.Barrier()
        secs[name] = round(time.time() - t0, 2)
    return {"checked": R.call, "by_part": R.done, "seconds": secs}


if __name__ == "__main__":
    opts, rest = parse_options(sys.argv[1:])
    sys.argv = [sys.argv[0]] + rest
    W.SCENARIOS["kinds"] = lambda a: scenario_kinds(a, opts)
    W.main()
