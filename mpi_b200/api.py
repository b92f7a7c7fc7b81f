"""Python mirror of the reference's package-level API (/root/reference/mpi.go:56-182).

Same names, same argument meaning, same blocking behaviour:

    Init() Finalize() Rank() Size() Send(data, destination, tag) Receive(data, source, tag)
    Register(impl)  Interface  Raw  TagExists                       (the reference's surface)
    Recv  Bcast(data, root)  Allreduce(send, recv, op)  Allgather(send, recv)  Barrier()   (new)
    ReduceScatter(send, recv, op)  Reduce(send, recv, op, root)  Alltoall(send, recv)      (new)
    Scan(send, recv, op)  Exscan(send, recv, op)                                             (new)
    Gather(send, recv, root)  Scatter(send, recv, root)                                       (new)
    Gatherv(send, recv, root, counts)  Scatterv(send, recv, counts, root)  Allgatherv(send, recv, counts)
    Alltoallv(send, send_counts, recv, recv_counts)                                          (new)
    ReduceScatterv(send, recv, counts, op)                                                   (new)
    AllreduceLoc(send, recv, op)  ReduceLoc(send, recv, op, root)   (MAXLOC / MINLOC, new)
    WinCreate(local) -> Win: Put, Get, Accumulate, Fence, Free      (one-sided, fence-synchronised, new)
        + Lock, Unlock, GetAccumulate, FetchAndOp, CompareAndSwap   (passive target, new)
        + Post, Start, Complete, Wait, Test                         (generalized active target, new)
    Isend(data, destination, tag) + Wait(destination, tag)     (the Send/Wait design commented out
                                                                in the reference, mpi.go:132-152)

Where Go returns `error`, Python raises MpiError (Go's "implementations may panic", mpi.go:20-21,
maps to the same exception).  `data` is type-switched exactly like the cgo shim
(go/mpi/cuda.go): float64 / float32 / int64 / uint8 numpy arrays and bytes-likes travel as typed
buffers; `str` is encoded to bytes first (the "anything else is gob-encoded" path of the reference);
DeviceSlice is memory from the library's device heap and takes the zero-copy path.
"""
import abc
import ctypes
import sys

import numpy as np

from . import _lib as L
from . import flags as _flags

SUM, MAX, MIN = L.SUM, L.MAX, L.MIN
REPLACE, NO_OP = L.REPLACE, L.NO_OP                      # one-sided only
LOCK_EXCLUSIVE, LOCK_SHARED = L.LOCK_EXCLUSIVE, L.LOCK_SHARED


class MpiError(Exception):
    def __init__(self, code, message):
        super().__init__("%s (b200mpi error %d)" % (message, code))
        self.code = code
        self.message = message


class TagExists(MpiError):
    """mpi.go:174-182: the tag already has a concurrent request between the two nodes."""

    def __init__(self, code, message, tag):
        super().__init__(code, message)
        self.Tag = tag


class Raw(bytes):
    """mpi.go:75: send as raw bytes, no encoding."""


_NP2DT = {np.dtype(np.uint8): L.U8, np.dtype(np.int64): L.I64, np.dtype(np.float32): L.F32, np.dtype(np.float64): L.F64}
_DT2NP = {v: k for k, v in _NP2DT.items()}

# The value-location pairs of AllreduceLoc / ReduceLoc: the C struct {V val; int64_t loc}, 16 bytes
# for every V (4 padding bytes after an f32 value).  Only those two calls take them.
LOC_F32 = np.dtype([("val", "<f4"), ("loc", "<i8")], align=True)
LOC_F64 = np.dtype([("val", "<f8"), ("loc", "<i8")], align=True)
LOC_I64 = np.dtype([("val", "<i8"), ("loc", "<i8")], align=True)
_LOC2DT = {LOC_F32: L.F32, LOC_F64: L.F64, LOC_I64: L.I64}


def _check(rc, tag=None):
    if rc == 0:
        return
    msg = L.last_error()
    if rc == L.ERR_TAG_EXISTS:
        raise TagExists(rc, msg, tag)
    raise MpiError(rc, msg)


class DeviceSlice:
    """`count` elements of `dtype` in this rank's peer-mapped device heap (b200mpi_alloc)."""

    def __init__(self, count, dtype, ptr=None, owner=True):
        self.dtype = np.dtype(dtype)
        if self.dtype not in _NP2DT and self.dtype not in _LOC2DT:
            raise TypeError("unsupported element type %s" % self.dtype)
        self.count = int(count)
        self._owner = owner
        if ptr is None:
            p = ctypes.c_void_p()
            _check(L.load().b200mpi_alloc(max(self.nbytes, 1), ctypes.byref(p)))
            ptr = p.value
        self.ptr = ptr

    @property
    def nbytes(self):
        return self.count * self.dtype.itemsize

    def __len__(self):
        return self.count

    def __getitem__(self, sl):
        if not isinstance(sl, slice):
            raise TypeError("DeviceSlice supports slicing only")
        start, stop, step = sl.indices(self.count)
        if step != 1:
            raise ValueError("DeviceSlice slices must be contiguous")
        return DeviceSlice(max(stop - start, 0), self.dtype, self.ptr + start * self.dtype.itemsize, owner=False)

    def copy_from_host(self, arr):
        a = np.ascontiguousarray(arr, dtype=self.dtype).reshape(-1)
        if a.size != self.count:
            raise ValueError("size mismatch: %d vs %d" % (a.size, self.count))
        if a.size:
            _check(L.load().b200mpi_memcpy(self.ptr, a.ctypes.data, a.nbytes, 0))
        return self

    def to_host(self):
        out = np.empty(self.count, dtype=self.dtype)
        if out.size:
            _check(L.load().b200mpi_memcpy(out.ctypes.data, self.ptr, out.nbytes, 1))
        return out

    def free(self):
        if self._owner and self.ptr:
            _check(L.load().b200mpi_free(self.ptr))
        self.ptr = None


def Alloc(count, dtype):
    return DeviceSlice(count, dtype)


def _describe(data):
    """-> (pointer, count, dtype code, memkind, keepalive, kind tag)."""
    if isinstance(data, DeviceSlice):
        if data.dtype not in _NP2DT:
            raise TypeError("mpi: value-location pairs (%s) go through AllreduceLoc and ReduceLoc only" % data.dtype)
        return data.ptr, data.count, _NP2DT[data.dtype], L.DEVICE, data, "device"
    if isinstance(data, np.ndarray):
        if data.dtype not in _NP2DT:
            raise TypeError("mpi: unsupported element type %s (want float64, float32, int64 or uint8)" % data.dtype)
        if not data.flags["C_CONTIGUOUS"]:
            raise ValueError("mpi: array must be contiguous")
        return (data.ctypes.data if data.size else None), data.size, _NP2DT[data.dtype], L.HOST, data, "ndarray"
    if isinstance(data, str):
        b = np.frombuffer(data.encode("utf-8"), dtype=np.uint8)
        return (b.ctypes.data if b.size else None), b.size, L.U8, L.HOST, b, "str"
    if isinstance(data, (bytes, bytearray, memoryview)):
        b = np.frombuffer(data, dtype=np.uint8)
        return (b.ctypes.data if b.size else None), b.size, L.U8, L.HOST, b, "bytes"
    raise TypeError("mpi: cannot send a %s" % type(data).__name__)


class Interface(abc.ABC):
    """mpi.go:163-170."""

    @abc.abstractmethod
    def Init(self): ...

    @abc.abstractmethod
    def Finalize(self): ...

    @abc.abstractmethod
    def Rank(self): ...

    @abc.abstractmethod
    def Size(self): ...

    @abc.abstractmethod
    def Send(self, data, destination, tag): ...

    @abc.abstractmethod
    def Receive(self, data, source, tag): ...


class Cuda(Interface):
    """The H100 implementation behind the facade; plays the role of `Network`
    (network.go:25-39): public fields win over flags (network.go:69-90)."""

    def __init__(self, Addr="", Addrs=None, Timeout=0, Password="", Gpu=None):
        self.Addr = Addr
        self.Addrs = list(Addrs) if Addrs else []
        self.Timeout = Timeout  # nanoseconds
        self.Password = Password
        self.Gpu = Gpu

    # -- lifecycle ---------------------------------------------------------------------------
    def _use_flags(self):
        f = _flags.parse(sys.argv[1:])
        if not self.Password:
            self.Password = f.password
        if not self.Timeout:
            self.Timeout = f.inittimeout
        if not self.Addr:
            self.Addr = f.addr
        if not self.Addrs:
            self.Addrs = list(f.alladdr)
        if self.Gpu is None:
            self.Gpu = f.gpu

    def Init(self):
        self._use_flags()
        lib = L.load()
        _check(lib.b200mpi_init(self.Addr.encode(), ",".join(self.Addrs).encode(), self.Password.encode(),
                                int(self.Timeout), int(-1 if self.Gpu is None else self.Gpu)))

    def Finalize(self):
        _check(L.load().b200mpi_finalize())

    def Rank(self):
        return L.load().b200mpi_rank()

    def Size(self):
        return L.load().b200mpi_size()

    # -- point to point ----------------------------------------------------------------------
    def Send(self, data, destination, tag):
        ptr, count, dt, kind, keep, _ = _describe(data)
        _check(L.load().b200mpi_send(ptr, count, dt, int(destination), int(tag), kind), tag)

    def Isend(self, data, destination, tag):
        """mpi.go:132-143 (commented design): returns once `data` may be modified again, without
        waiting for the receiver; Wait(destination, tag) collects the confirmation."""
        ptr, count, dt, kind, keep, _ = _describe(data)
        _check(L.load().b200mpi_isend(ptr, count, dt, int(destination), int(tag), kind), tag)

    def Wait(self, destination, tag):
        """mpi.go:146-152 (commented design)."""
        _check(L.load().b200mpi_wait(int(destination), int(tag)), tag)

    def Receive(self, data, source, tag):
        """Fills `data` and returns the received value.  numpy arrays and bytearrays are filled
        in place when large enough (a view of the received length is returned), otherwise a new
        object of the sent length is returned -- the analogue of gob resizing the destination
        slice (network.go:597).  Pass the type `str` / `bytes` (or an instance) to receive one."""
        lib = L.load()
        n = ctypes.c_size_t(0)
        if isinstance(data, DeviceSlice):
            _, _, dt, _, _, _ = _describe(data)
            _check(lib.b200mpi_recv(data.ptr, data.count, ctypes.byref(n), dt, int(source), int(tag), L.DEVICE), tag)
            return data[: n.value]
        want_str = data is str or isinstance(data, str)
        want_bytes = data is bytes or isinstance(data, bytes)
        if want_str or want_bytes:
            buf = np.empty(256, dtype=np.uint8)
        elif isinstance(data, bytearray):
            buf = np.frombuffer(data, dtype=np.uint8) if len(data) else np.empty(0, dtype=np.uint8)
        elif isinstance(data, np.ndarray):
            if data.dtype not in _NP2DT:
                raise TypeError("mpi: unsupported element type %s" % data.dtype)
            buf = data.reshape(-1)
        else:
            raise TypeError("mpi: cannot receive into a %s" % type(data).__name__)
        dt = _NP2DT[buf.dtype]
        rc = lib.b200mpi_recv(buf.ctypes.data if buf.size else None, buf.size, ctypes.byref(n), dt, int(source), int(tag), L.HOST)
        if rc == L.ERR_TRUNCATE:  # message is still posted: retry with the right size
            buf = np.empty(n.value, dtype=buf.dtype)
            rc = lib.b200mpi_recv(buf.ctypes.data, buf.size, ctypes.byref(n), dt, int(source), int(tag), L.HOST)
            if isinstance(data, bytearray) and rc == 0:
                data[:] = buf.tobytes()
                return data
        _check(rc, tag)
        out = buf[: n.value]
        if want_str:
            return out.tobytes().decode("utf-8")
        if want_bytes:
            return out.tobytes()
        if isinstance(data, bytearray):
            del data[n.value:]
            return data
        return out

    # -- collectives (the optional upgrade interface hinted at by mpi.go:69-71) ---------------
    def Bcast(self, data, root):
        ptr, count, dt, kind, keep, tagk = _describe(data)
        if tagk in ("str", "bytes") and not isinstance(data, (bytearray, memoryview)):
            raise TypeError("mpi: Bcast needs a mutable buffer (numpy array, bytearray or DeviceSlice)")
        _check(L.load().b200mpi_bcast(ptr, count, dt, int(root), kind))
        return data

    def Allreduce(self, send, recv, op=SUM):
        sp, sc, sdt, sk, _, _ = _describe(send)
        rp, rc_, rdt, rk, _, _ = _describe(recv)
        if sc != rc_ or sdt != rdt or sk != rk:
            raise ValueError("mpi: Allreduce send and recv must have the same length, type and memory kind")
        _check(L.load().b200mpi_allreduce(sp, rp, sc, sdt, int(op), sk))
        return recv

    def Allgather(self, send, recv):
        sp, sc, sdt, sk, _, _ = _describe(send)
        rp, rc_, rdt, rk, _, _ = _describe(recv)
        if rc_ != sc * self.Size() or sdt != rdt or sk != rk:
            raise ValueError("mpi: Allgather recv must hold Size()*len(send) elements of the same type and memory kind")
        _check(L.load().b200mpi_allgather(sp, rp, sc, sdt, sk))
        return recv

    def ReduceScatter(self, send, recv, op=SUM):
        sp, sc, sdt, sk, _, _ = _describe(send)
        rp, rc_, rdt, rk, _, _ = _describe(recv)
        if sc != rc_ * self.Size() or sdt != rdt or sk != rk:
            raise ValueError("mpi: ReduceScatter send must hold Size()*len(recv) elements of the same type and memory kind")
        _check(L.load().b200mpi_reduce_scatter(sp, rp, rc_, sdt, int(op), sk))
        return recv

    def Reduce(self, send, recv, op=SUM, root=0):
        sp, sc, sdt, sk, _, _ = _describe(send)
        if recv is None:
            rp = None
        else:
            rp, rc_, rdt, rk, _, _ = _describe(recv)
            if sc != rc_ or sdt != rdt or sk != rk:
                raise ValueError("mpi: Reduce send and recv must have the same length, type and memory kind")
        _check(L.load().b200mpi_reduce(sp, rp, sc, sdt, int(op), int(root), sk))
        return recv

    def Alltoall(self, send, recv):
        sp, sc, sdt, sk, _, _ = _describe(send)
        rp, rc_, rdt, rk, _, _ = _describe(recv)
        n = self.Size()
        if sc != rc_ or sc % max(n, 1) or sdt != rdt or sk != rk:
            raise ValueError("mpi: Alltoall send and recv must both hold Size() equal blocks of the same type and memory kind")
        _check(L.load().b200mpi_alltoall(sp, rp, sc // n, sdt, sk))
        return recv

    def Scan(self, send, recv, op=SUM):
        """Rank r's recv = send_0 op ... op send_r, combined in rank order.  recv is send: in place."""
        sp, sc, sdt, sk, _, _ = _describe(send)
        rp, rc_, rdt, rk, _, _ = _describe(recv)
        if sc != rc_ or sdt != rdt or sk != rk:
            raise ValueError("mpi: Scan send and recv must have the same length, type and memory kind")
        _check(L.load().b200mpi_scan(sp, rp, sc, sdt, int(op), sk))
        return recv

    def Exscan(self, send, recv, op=SUM):
        """Rank r's recv = send_0 op ... op send_{r-1}; rank 0's recv is not written and may be None
        there (the library refuses None elsewhere)."""
        sp, sc, sdt, sk, _, _ = _describe(send)
        rp = None
        if recv is not None:
            rp, rc_, rdt, rk, _, _ = _describe(recv)
            if sc != rc_ or sdt != rdt or sk != rk:
                raise ValueError("mpi: Exscan send and recv must have the same length, type and memory kind")
        _check(L.load().b200mpi_exscan(sp, rp, sc, sdt, int(op), sk))
        return recv

    def Barrier(self):
        _check(L.load().b200mpi_barrier())

    # -- rooted and variable-count collectives ----------------------------------------------------
    def _world(self):
        n = self.Size()
        if n <= 0:
            raise MpiError(L.ERR_NOT_INIT, "mpi: Init has not been called")
        return self.Rank(), n

    def Gather(self, send, recv, root):
        """Rank r's send lands in block r of root's recv (Size()*len(send) elements); recv is
        ignored and may be None off root.  In place on root: send is root's block of recv."""
        rank, n = self._world()
        sp, sc, sdt, sk, keep, _ = _describe(send)  # keep: a str travels as a temporary encoding
        rp = None
        if rank == root:
            if recv is None:
                raise ValueError("mpi: Gather needs a recv buffer on root")
            rp, rc_, rdt, rk, _, _ = _describe(recv)
            if rc_ != sc * n or sdt != rdt or sk != rk:
                raise ValueError("mpi: Gather recv must hold Size()*len(send) elements of the same type and memory kind")
        _check(L.load().b200mpi_gather(sp, rp, sc, sdt, int(root), sk))
        return recv

    def Scatter(self, send, recv, root):
        """Block r of root's send (Size()*len(recv) elements) goes to rank r's recv; send is
        ignored and may be None off root.  In place on root: recv is root's block of send."""
        rank, n = self._world()
        rp, rc_, rdt, rk, _, _ = _describe(recv)
        sp = None
        if rank == root:
            if send is None:
                raise ValueError("mpi: Scatter needs a send buffer on root")
            sp, sc, sdt, sk, keep, _ = _describe(send)
            if sc != rc_ * n or sdt != rdt or sk != rk:
                raise ValueError("mpi: Scatter send must hold Size()*len(recv) elements of the same type and memory kind")
        _check(L.load().b200mpi_scatter(sp, rp, rc_, rdt, int(root), rk))
        return recv

    def _table(self, counts, n):
        counts = [int(c) for c in counts]
        if len(counts) != n or any(c < 0 for c in counts):
            raise ValueError("mpi: counts must hold Size() non-negative element counts")
        return counts, (ctypes.c_size_t * n)(*counts)

    def _lengths(self, count):
        """Every rank's element count, through one int64 Allgather."""
        n = self.Size()
        mine = np.array([count], dtype=np.int64)
        everyone = np.empty(n, dtype=np.int64)
        self.Allgather(mine, everyone)
        return everyone.tolist()

    @staticmethod
    def _recv_for(recv, total, dt, kind, what):
        """recv of `total` elements: a host array that is missing or too small is replaced by a new one
        (as Receive resizes), a larger one is used through a view of the right length."""
        if recv is None:
            if kind != L.HOST:
                raise ValueError("mpi: %s needs a recv DeviceSlice for a DeviceSlice send" % what)
            recv = np.empty(total, dtype=_DT2NP[dt])
        rp, rc_, rdt, rk, _, _ = _describe(recv)
        if rdt != dt or rk != kind:
            raise ValueError("mpi: %s send and recv must have the same type and memory kind" % what)
        if rc_ != total:
            if rk != L.HOST or not isinstance(recv, np.ndarray):
                raise ValueError("mpi: %s recv must hold %d elements" % (what, total))
            recv = np.empty(total, dtype=_DT2NP[dt]) if rc_ < total else recv.reshape(-1)[:total]
            rp = recv.ctypes.data if total else None
        return recv, rp

    def Gatherv(self, send, recv=None, root=0, counts=None):
        """Rank r's send lands at displacement counts[0]+...+counts[r-1] of root's recv.  counts is
        the same table on every rank; omitted on every rank, it is learnt with one Allgather.
        Returns (recv, counts); off root recv is returned as passed."""
        rank, n = self._world()
        sp, sc, sdt, sk, keep, _ = _describe(send)
        if counts is None:
            counts = self._lengths(sc)
        counts, table = self._table(counts, n)
        if counts[rank] != sc:
            raise ValueError("mpi: Gatherv counts[Rank()] must equal len(send)")
        rp = None
        if rank == root:
            recv, rp = self._recv_for(recv, sum(counts), sdt, sk, "Gatherv")
        _check(L.load().b200mpi_gatherv(sp, rp, table, sdt, int(root), sk))
        return recv, counts

    def Allgatherv(self, send, recv=None, counts=None):
        """Rank r's send lands at displacement counts[0]+...+counts[r-1] of every rank's recv.
        counts as for Gatherv.  Returns (recv, counts)."""
        rank, n = self._world()
        sp, sc, sdt, sk, keep, _ = _describe(send)
        if counts is None:
            counts = self._lengths(sc)
        counts, table = self._table(counts, n)
        if counts[rank] != sc:
            raise ValueError("mpi: Allgatherv counts[Rank()] must equal len(send)")
        recv, rp = self._recv_for(recv, sum(counts), sdt, sk, "Allgatherv")
        _check(L.load().b200mpi_allgatherv(sp, rp, table, sdt, sk))
        return recv, counts

    def Scatterv(self, send, recv, counts=None, root=0):
        """Block r of root's send, at displacement counts[0]+...+counts[r-1], goes to rank r's recv.
        Root passes counts; the other ranks may pass None and learn root's table, which root always
        sends with one small Bcast.  A host recv that is too small is replaced as in Gatherv; recv
        gives the element type, so it is needed on every rank.  Returns (recv, counts)."""
        rank, n = self._world()
        if recv is None:
            raise ValueError("mpi: Scatterv needs a recv buffer (or an empty array of the element type)")
        _, rc_, rdt, rk, _, _ = _describe(recv)
        sp = None
        if rank == root:
            if send is None or counts is None:
                raise ValueError("mpi: Scatterv needs send and counts on root")
            sp, sc, sdt, sk, keep, _ = _describe(send)
            counts, _ = self._table(counts, n)
            if sum(counts) != sc or sdt != rdt or sk != rk:
                raise ValueError("mpi: Scatterv send must hold sum(counts) elements of recv's type and memory kind")
        elif counts is not None:
            counts, _ = self._table(counts, n)
        root_table = np.array(counts if rank == root else [0] * n, dtype=np.int64)
        self.Bcast(root_table, root)
        if counts is None:
            counts = root_table.tolist()
        counts, table = self._table(counts, n)  # a table that differs from root's fails as ERR_PEER on every rank
        recv, rp = self._recv_for(recv, counts[rank], rdt, rk, "Scatterv")
        _check(L.load().b200mpi_scatterv(sp, rp, table, rdt, int(root), rk))
        return recv, counts

    def Alltoallv(self, send, send_counts, recv=None, recv_counts=None):
        """Block j of send (send_counts[j] elements, packed in rank order) goes to rank j; the block
        from rank r lands at displacement recv_counts[0]+...+recv_counts[r-1] of recv.  recv_counts[r]
        must equal rank r's send_counts[Rank()]; omitted, it is learnt with one int64 Alltoall of
        send_counts.  A host recv is created or resized as in Gatherv.  Returns (recv, recv_counts)."""
        rank, n = self._world()
        sp, sc, sdt, sk, keep, _ = _describe(send)
        send_counts, stable = self._table(send_counts, n)
        if sum(send_counts) != sc:
            raise ValueError("mpi: Alltoallv send must hold sum(send_counts) elements")
        if recv_counts is None:
            learnt = np.empty(n, dtype=np.int64)
            self.Alltoall(np.array(send_counts, dtype=np.int64), learnt)
            recv_counts = learnt.tolist()
        recv_counts, rtable = self._table(recv_counts, n)
        recv, rp = self._recv_for(recv, sum(recv_counts), sdt, sk, "Alltoallv")
        _check(L.load().b200mpi_alltoallv(sp, stable, rp, rtable, sdt, sk))
        return recv, recv_counts

    def ReduceScatterv(self, send, recv=None, counts=None, op=SUM):
        """Rank j's recv receives op over every rank's block j, combined in rank order; block j is
        counts[j] elements at displacement counts[0]+...+counts[j-1] of send (sum(counts) elements).
        counts is the same table on every rank; omitted on every rank, it is learnt from len(recv)
        with one Allgather.  A host recv is created or resized as in Gatherv.  In place: recv is
        this rank's block of send.  Returns (recv, counts)."""
        rank, n = self._world()
        sp, sc, sdt, sk, keep, _ = _describe(send)
        if counts is None:
            if recv is None:
                raise ValueError("mpi: ReduceScatterv needs counts or a recv to learn them from")
            counts = self._lengths(_describe(recv)[1])
        counts, table = self._table(counts, n)
        if sum(counts) != sc:
            raise ValueError("mpi: ReduceScatterv send must hold sum(counts) elements")
        recv, rp = self._recv_for(recv, counts[rank], sdt, sk, "ReduceScatterv")
        _check(L.load().b200mpi_reduce_scatterv(sp, rp, table, sdt, int(op), sk))
        return recv, counts

    @staticmethod
    def _describe_loc(data, what):
        """-> (pointer, count, value dtype code, memkind) of a pair array or DeviceSlice."""
        if isinstance(data, DeviceSlice):
            dt, ptr, kind = data.dtype, data.ptr, L.DEVICE
        elif isinstance(data, np.ndarray):
            if not data.flags["C_CONTIGUOUS"]:
                raise ValueError("mpi: array must be contiguous")
            dt, ptr, kind = data.dtype, (data.ctypes.data if data.size else None), L.HOST
        else:
            raise TypeError("mpi: %s takes a numpy array or DeviceSlice of pairs, not a %s" % (what, type(data).__name__))
        if dt not in _LOC2DT:
            raise TypeError("mpi: %s needs value-location pairs (LOC_F32, LOC_F64 or LOC_I64), not %s" % (what, dt))
        return ptr, len(data), _LOC2DT[dt], kind

    def AllreduceLoc(self, send, recv, op=MAX):
        """MAXLOC (op MAX) / MINLOC (op MIN) over {val, loc} pairs, combined in rank order: a higher
        rank's pair wins when its value is better, or equal with a smaller loc; NaN beats every number
        under both ops.  Every rank's recv gets the winning pairs whole.  recv is send: in place."""
        sp, sc, sdt, sk = self._describe_loc(send, "AllreduceLoc")
        rp, rc_, rdt, rk = self._describe_loc(recv, "AllreduceLoc")
        if sc != rc_ or sdt != rdt or sk != rk:
            raise ValueError("mpi: AllreduceLoc send and recv must have the same length, pair type and memory kind")
        _check(L.load().b200mpi_allreduce_loc(sp, rp, sc, sdt, int(op), sk))
        return recv

    def ReduceLoc(self, send, recv, op=MAX, root=0):
        """AllreduceLoc whose result lands in root's recv only; recv may be None elsewhere."""
        sp, sc, sdt, sk = self._describe_loc(send, "ReduceLoc")
        rp = None
        if recv is not None:
            rp, rc_, rdt, rk = self._describe_loc(recv, "ReduceLoc")
            if sc != rc_ or sdt != rdt or sk != rk:
                raise ValueError("mpi: ReduceLoc send and recv must have the same length, pair type and memory kind")
        _check(L.load().b200mpi_reduce_loc(sp, rp, sc, sdt, int(op), int(root), sk))
        return recv


    # -- one-sided communication ----------------------------------------------------------------
    def WinCreate(self, local):
        """Collective: exposes `local`, a DeviceSlice from Alloc (or None for an empty window), to
        one-sided Put, Get and Accumulate by every rank.  Windows may differ in size from rank to rank."""
        if local is None:
            ptr, nbytes = None, 0
        elif isinstance(local, DeviceSlice):
            ptr, nbytes = local.ptr, local.nbytes
        else:
            raise TypeError("mpi: a window is a DeviceSlice from Alloc (or None), not a %s" % type(local).__name__)
        wid = ctypes.c_int(-1)
        _check(L.load().b200mpi_win_create(ptr, nbytes, ctypes.byref(wid)))
        return Win(wid.value)


class Win:
    """A window of every rank's heap (WinCreate).  Put, Get and Accumulate move the origin's elements
    to or from element `disp` of rank `target`'s window, counted in the origin's element type, and
    block until the origin may be reused (Get: until it holds the data).  What they write is visible
    to the target after its next Fence, which every rank calls; a location written by one rank and
    read or written by another between two fences is undefined, except by Accumulates with the same
    type and op.  Free is a Fence that also drops the window.

    Passive target: Lock(target) / Unlock(target) give this rank mutual exclusion on one target's
    window without the other ranks taking part; every call has completed when it returns, so what a
    rank did under the lock is visible to the next holder.  GetAccumulate, FetchAndOp and
    CompareAndSwap return the target's previous values, one atomic per element.  A rank holding a lock
    on this window must not Fence or Free it (MpiError, and the other ranks' call fails too).

    Generalized active target: a target calls Post(origins) to expose its window to a group of ranks
    and Wait() (or Test()) to close that epoch; an origin calls Start(targets), which blocks until each
    target has posted to it, and Complete() once its Put, Get and Accumulate calls are done.  Only the
    ranks in the groups take part.  What the origins put between Start and Complete is visible to the
    target once its Wait returns.  A group is an iterable of distinct ranks (Python or numpy ints),
    possibly empty or containing this rank.  A rank with an epoch open on this window must not Fence
    or Free it, as under a lock."""

    def __init__(self, wid):
        self.id = wid

    @staticmethod
    def _origin(origin, disp, what):
        """-> (pointer, count, dtype code, memkind); refuses pairs and negative displacements."""
        ptr, count, dt, kind, _, _ = _describe(origin)
        if int(disp) < 0:
            raise ValueError("mpi: %s displacement must be >= 0" % what)
        return ptr, count, dt, kind

    def Put(self, origin, target, disp=0):
        ptr, count, dt, kind = self._origin(origin, disp, "Put")
        _check(L.load().b200mpi_put(ptr, count, dt, int(target), int(disp), self.id, kind))

    def Get(self, origin, target, disp=0):
        """Fills `origin` (a numpy array, bytearray or DeviceSlice) from the target's window and returns it."""
        if (isinstance(origin, (str, bytes)) or (isinstance(origin, memoryview) and origin.readonly)
                or (isinstance(origin, np.ndarray) and not origin.flags["WRITEABLE"])):
            raise TypeError("mpi: Get needs a writable buffer (numpy array, bytearray or DeviceSlice)")
        ptr, count, dt, kind = self._origin(origin, disp, "Get")
        _check(L.load().b200mpi_get(ptr, count, dt, int(target), int(disp), self.id, kind))
        return origin

    def Accumulate(self, origin, target, disp=0, op=SUM):
        """target[disp + i] = target[disp + i] op origin[i], element by element and atomically, for
        float32, float64 and int64 (an f32 SUM flushes subnormals to zero; see b200mpi.h)."""
        ptr, count, dt, kind = self._origin(origin, disp, "Accumulate")
        _check(L.load().b200mpi_accumulate(ptr, count, dt, int(op), int(target), int(disp), self.id, kind))

    def Lock(self, target, lock_type=LOCK_EXCLUSIVE):
        """Blocks until this rank holds the lock on rank `target`'s window (LOCK_EXCLUSIVE or
        LOCK_SHARED); MpiError ERR_TIMEOUT if it is not granted within the watchdog_ms knob."""
        if lock_type not in (LOCK_EXCLUSIVE, LOCK_SHARED):
            raise ValueError("mpi: lock_type must be LOCK_EXCLUSIVE or LOCK_SHARED")
        _check(L.load().b200mpi_win_lock(int(lock_type), int(target), self.id))

    def Unlock(self, target):
        _check(L.load().b200mpi_win_unlock(int(target), self.id))

    def GetAccumulate(self, origin, result, target, disp=0, op=SUM):
        """result[i] = target[disp + i] before, then target[disp + i] = target[disp + i] op origin[i],
        element by element and atomically; op SUM, MAX, MIN, REPLACE or NO_OP (origin may be None).
        result has origin's element type, length and storage (it may be origin itself); returns it."""
        if (isinstance(result, (str, bytes)) or (isinstance(result, memoryview) and result.readonly)
                or (isinstance(result, np.ndarray) and not result.flags["WRITEABLE"])):
            raise TypeError("mpi: GetAccumulate needs a writable result (numpy array, bytearray or DeviceSlice)")
        rptr, count, dt, kind = self._origin(result, disp, "GetAccumulate")
        optr = None
        if origin is not None:
            optr, ocount, odt, okind = self._origin(origin, disp, "GetAccumulate")
            if odt != dt or okind != kind:
                raise TypeError("mpi: GetAccumulate's origin and result must have one element type and storage")
            if ocount != count:
                raise ValueError("mpi: GetAccumulate's origin and result must have the same length")
        elif int(op) != NO_OP:
            raise TypeError("mpi: GetAccumulate needs an origin unless op is NO_OP")
        _check(L.load().b200mpi_get_accumulate(optr, rptr, count, dt, int(op), int(target), int(disp), self.id, kind))
        return result

    @staticmethod
    def _scalar(value, what, allowed=(np.float32, np.float64, np.int64)):
        """A one-element array of the value's numpy type (int: int64, float: float64)."""
        if isinstance(value, (bool, np.bool_)):
            raise TypeError("mpi: %s takes a number, not a bool" % what)
        if isinstance(value, int):
            value = np.int64(value)
        elif isinstance(value, float):
            value = np.float64(value)
        if not isinstance(value, allowed):
            raise TypeError("mpi: %s takes %s, not %s" % (what, " / ".join(t.__name__ for t in allowed), type(value).__name__))
        return np.array([value], dtype=type(value))

    def FetchAndOp(self, value, target, disp=0, op=SUM):
        """One element: returns target[disp] before, then target[disp] = target[disp] op value, atomically.
        value is an np.float32, np.float64 or np.int64 (int: int64, float: float64); the result has its type."""
        v = self._scalar(value, "FetchAndOp")
        if int(disp) < 0:
            raise ValueError("mpi: FetchAndOp displacement must be >= 0")
        res = np.zeros(1, dtype=v.dtype)
        optr = None if int(op) == NO_OP else v.ctypes.data
        _check(L.load().b200mpi_fetch_and_op(optr, res.ctypes.data, _NP2DT[v.dtype], int(op), int(target), int(disp), self.id))
        return res[0]

    def CompareAndSwap(self, value, compare, target, disp=0):
        """int64: returns target[disp] before, and stores value there if that equals compare, atomically."""
        v = self._scalar(value, "CompareAndSwap", (np.int64,))
        c = self._scalar(compare, "CompareAndSwap", (np.int64,))
        if int(disp) < 0:
            raise ValueError("mpi: CompareAndSwap displacement must be >= 0")
        res = np.zeros(1, dtype=np.int64)
        _check(L.load().b200mpi_compare_and_swap(v.ctypes.data, c.ctypes.data, res.ctypes.data, L.I64, int(target), int(disp), self.id))
        return res[0]

    @staticmethod
    def _group(ranks, what):
        """A C int array of the ranks of an iterable of Python or numpy ints (range and duplicates are
        the library's to check) and its length."""
        try:
            items = list(ranks)
        except TypeError:
            raise TypeError("mpi: %s takes an iterable of ranks, not %s" % (what, type(ranks).__name__)) from None
        for r in items:
            if isinstance(r, (bool, np.bool_)) or not isinstance(r, (int, np.integer)):
                raise TypeError("mpi: %s takes ranks as ints, not %s" % (what, type(r).__name__))
        arr = (ctypes.c_int * max(len(items), 1))()
        for i, r in enumerate(items):
            arr[i] = int(r) if -2**31 <= int(r) < 2**31 else -1  # -1: out of range, which the library refuses
        return arr, len(items)

    def Post(self, origins):
        """Opens an exposure epoch of this window to the ranks in `origins`; does not block."""
        arr, n = self._group(origins, "Post")
        _check(L.load().b200mpi_win_post(arr, n, self.id))

    def Start(self, targets):
        """Opens an access epoch to the ranks in `targets`: blocks until each has posted to this rank
        (MpiError ERR_TIMEOUT, and no epoch open, if one has not within the watchdog_ms knob)."""
        arr, n = self._group(targets, "Start")
        _check(L.load().b200mpi_win_start(arr, n, self.id))

    def Complete(self):
        """Closes the access epoch: tells each target of Start that this rank is done."""
        _check(L.load().b200mpi_win_complete(self.id))

    def Wait(self):
        """Closes the exposure epoch once every origin of Post has called Complete (MpiError
        ERR_TIMEOUT, the epoch still open, if they have not within the watchdog_ms knob)."""
        _check(L.load().b200mpi_win_wait(self.id))

    def Test(self):
        """Wait without waiting: True and the exposure epoch closed, or False and still open."""
        flag = ctypes.c_int(0)
        _check(L.load().b200mpi_win_test(self.id, ctypes.byref(flag)))
        return bool(flag.value)

    def Fence(self):
        _check(L.load().b200mpi_win_fence(self.id))

    def Free(self):
        _check(L.load().b200mpi_win_free(self.id))


# ---- package-level facade: mpi.go:56-159 -------------------------------------------------------
_mpier = Cuda()
_register_called = False


def Register(impl):
    """mpi.go:61-67: install an implementation; a second call panics."""
    global _mpier, _register_called
    _mpier = impl
    if _register_called:
        raise RuntimeError("register called more than once")
    _register_called = True


def _reset_for_tests(impl=None):
    global _mpier, _register_called
    _mpier = impl if impl is not None else Cuda()
    _register_called = False


def Init():
    return _mpier.Init()


def Finalize():
    return _mpier.Finalize()


def Rank():
    return _mpier.Rank()


def Size():
    return _mpier.Size()


def Send(data, destination, tag):
    return _mpier.Send(data, destination, tag)


def Receive(data, source, tag):
    return _mpier.Receive(data, source, tag)


Recv = Receive  # north_star spells it Recv; the reference spells it Receive (mpi.go:157)


def _collective(name):
    fn = getattr(_mpier, name, None)
    if fn is None:
        raise MpiError(L.ERR_UNSUPPORTED, "registered implementation has no %s" % name)
    return fn


def Bcast(data, root):
    return _collective("Bcast")(data, root)


def Allreduce(send, recv, op=SUM):
    return _collective("Allreduce")(send, recv, op)


def Allgather(send, recv):
    return _collective("Allgather")(send, recv)


def Barrier():
    return _collective("Barrier")()


def ReduceScatter(send, recv, op=SUM):
    return _collective("ReduceScatter")(send, recv, op)


def Reduce(send, recv, op=SUM, root=0):
    return _collective("Reduce")(send, recv, op, root)


def Alltoall(send, recv):
    return _collective("Alltoall")(send, recv)


def Scan(send, recv, op=SUM):
    return _collective("Scan")(send, recv, op)


def Exscan(send, recv, op=SUM):
    return _collective("Exscan")(send, recv, op)


def Gather(send, recv, root):
    return _collective("Gather")(send, recv, root)


def Scatter(send, recv, root):
    return _collective("Scatter")(send, recv, root)


def Gatherv(send, recv=None, root=0, counts=None):
    return _collective("Gatherv")(send, recv, root, counts)


def Scatterv(send, recv, counts=None, root=0):
    return _collective("Scatterv")(send, recv, counts, root)


def Allgatherv(send, recv=None, counts=None):
    return _collective("Allgatherv")(send, recv, counts)


def Alltoallv(send, send_counts, recv=None, recv_counts=None):
    return _collective("Alltoallv")(send, send_counts, recv, recv_counts)


def ReduceScatterv(send, recv=None, counts=None, op=SUM):
    return _collective("ReduceScatterv")(send, recv, counts, op)


def AllreduceLoc(send, recv, op=MAX):
    return _collective("AllreduceLoc")(send, recv, op)


def ReduceLoc(send, recv, op=MAX, root=0):
    return _collective("ReduceLoc")(send, recv, op, root)


def WinCreate(local):
    return _collective("WinCreate")(local)


def Isend(data, destination, tag):
    return _collective("Isend")(data, destination, tag)


def Wait(destination, tag):
    return _collective("Wait")(destination, tag)
