"""One rank of a test world for AllreduceLoc and ReduceLoc (MAXLOC / MINLOC).  Usage as _worker.py:
_loc_worker.py <scenario> --out FILE [scenario args] -mpi-* flags.  Every buffer is a guarded view
(_kinds_worker.Buf: heap, device memory outside the heap, pinned or pageable host memory) and every
call is checked over the whole allocation: the destination holds the C oracle's pairs byte for byte,
padding included, and every guard and every buffer the call must not write is unchanged."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _footprint_worker as F  # noqa: E402
import _kinds_worker as K  # noqa: E402
import _loc_oracle as LO  # noqa: E402
import _loc_ref as R  # noqa: E402
import _worker as W  # noqa: E402
from _worker import L, mpi  # noqa: E402

DNS = ("f32", "f64", "i64")
OPS = (("maxloc", mpi.MAX), ("minloc", mpi.MIN))
STORAGES = ("heap", "torch", "pinned", "pageable")
CODE = {"f32": L.F32, "f64": L.F64, "i64": L.I64}
MANY_BLOCKS = 100003  # pairs; with own_block_bytes 4096 (256 pairs a block) about 390 ownership blocks


class World:
    def __init__(self):
        self.lib = L.load()
        self.rank, self.n = mpi.Rank(), mpi.Size()
        self.call = 0

    def next_call(self):
        self.call += 2
        return self.call


def loc_call(Wd, dn, opname, count, storage, layout, inplace=False, root=None, facade=False, null_recv=False):
    """One AllreduceLoc (root None) or ReduceLoc on guarded buffers, checked against the oracle.  In
    place: recv is send.  null_recv: a ReduceLoc off root passes NULL (None) as recv."""
    lib, rank, n = Wd.lib, Wd.rank, Wd.n
    op = dict(OPS)[opname]
    call = Wd.next_call()
    dt = R.LOC[dn]
    ins = R.tie_heavy(dn, n, count, call)
    offs = F.layout_offsets(layout, np.float64, n, call)  # byte residues 0 and 8 mod 16
    send = K.Buf(storage, dt, count, offs[rank][0], rank, call, body=ins[rank])
    gets = root is None or rank == root
    recv = None
    if not inplace and not (null_recv and not gets):
        recv = K.Buf(storage, dt, count, offs[rank][1], rank, call + 1)
    what = "%s dtype=%s op=%s count=%d storage=%s layout=%s offsets=%s inplace=%s root=%s facade=%s null_recv=%s rank=%d n=%d" % (
        "allreduce_loc" if root is None else "reduce_loc", dn, opname, count, storage, layout, offs, inplace, root, facade, null_recv, rank, n)
    W.trace(what)
    if facade:
        rv = send.view if inplace else (recv.view if recv is not None else None)
        if root is None:
            assert mpi.AllreduceLoc(send.view, rv, op) is rv
        else:
            mpi.ReduceLoc(send.view, rv, op, root)
    else:
        sp = send.ptr()
        rp = sp if inplace else (recv.ptr() if recv is not None else None)
        if root is None:
            rc = lib.b200mpi_allreduce_loc(sp, rp, count, CODE[dn], op, send.memkind)
        else:
            rc = lib.b200mpi_reduce_loc(sp, rp, count, CODE[dn], op, root, send.memkind)
        assert rc == 0, (what, rc, L.last_error())
    want = LO.allreduce_loc(ins, op)
    assert R.same(want, R.allreduce_loc_np(ins, op)), what
    if inplace:
        if gets:
            send.set_body(want)
        F.check(send, what + " [in-place buffer]")
    else:
        F.check(send, what + " [send must be unchanged]")
        if recv is not None:
            if gets:
                recv.set_body(want)
            F.check(recv, what + (" [recv]" if gets else " [recv off root must be unchanged]"))
            recv.free()
    send.free()
    return 1


def argument_errors(Wd):
    """Refusals, each the same on every rank, before anything is launched."""
    lib = Wd.lib
    a = mpi.Alloc(64, np.uint8)
    p = a.ptr
    cases = (
        ("u8 values", lambda: lib.b200mpi_allreduce_loc(p, p, 1, L.U8, L.MAX, L.DEVICE), L.ERR_UNSUPPORTED),
        ("op sum", lambda: lib.b200mpi_allreduce_loc(p, p, 1, L.F64, L.SUM, L.DEVICE), L.ERR_UNSUPPORTED),
        ("op sum (reduce_loc)", lambda: lib.b200mpi_reduce_loc(p, p, 1, L.I64, L.SUM, 0, L.DEVICE), L.ERR_UNSUPPORTED),
        ("unknown dtype", lambda: lib.b200mpi_allreduce_loc(p, p, 1, 9, L.MAX, L.DEVICE), L.ERR_UNSUPPORTED),
        ("unknown op", lambda: lib.b200mpi_allreduce_loc(p, p, 1, L.F32, 7, L.DEVICE), L.ERR_ARG),
        ("root out of range", lambda: lib.b200mpi_reduce_loc(p, p, 1, L.F32, L.MIN, Wd.n, L.DEVICE), L.ERR_ARG),
        ("negative root", lambda: lib.b200mpi_reduce_loc(p, p, 1, L.F32, L.MIN, -1, L.DEVICE), L.ERR_ARG),
        ("bad memkind", lambda: lib.b200mpi_allreduce_loc(p, p, 1, L.F32, L.MIN, 5), L.ERR_ARG),
        ("NULL send", lambda: lib.b200mpi_allreduce_loc(None, p, 1, L.F64, L.MAX, L.DEVICE), L.ERR_ARG),
        ("NULL recv", lambda: lib.b200mpi_allreduce_loc(p, None, 1, L.F64, L.MAX, L.DEVICE), L.ERR_ARG),
        ("send 4 mod 8", lambda: lib.b200mpi_allreduce_loc(p + 4, p + 32, 1, L.F64, L.MAX, L.DEVICE), L.ERR_ARG),
        ("recv 4 mod 8", lambda: lib.b200mpi_allreduce_loc(p, p + 20, 1, L.I64, L.MAX, L.DEVICE), L.ERR_ARG),
    )
    done = 0
    for name, call, want in cases:
        rc = call()
        assert rc == want, (name, rc, want, L.last_error())
        done += 1
    # count 0 with NULL buffers is legal, and a NULL recv off root
    assert lib.b200mpi_allreduce_loc(None, None, 0, L.F32, L.MAX, L.HOST) == 0, L.last_error()
    assert lib.b200mpi_reduce_loc(None, None, 0, L.I64, L.MIN, Wd.n - 1, L.DEVICE) == 0, L.last_error()
    a.free()
    return done + 2


def scenario_loc(a):
    """Argument errors; then every dtype, op and storage at counts 0, 1, 2, 3, 255 and one spanning
    many ownership blocks, AllreduceLoc in and out of place, at the four layouts of
    _footprint_worker.py (heap views at 8 mod 16 take the element path); then ReduceLoc at every root,
    with a NULL recv off root on every other call."""
    Wd = World()
    n = Wd.n
    done = argument_errors(Wd)
    counts = (0, 1, 2, 3, 255, MANY_BLOCKS)
    i = 0
    for dn in DNS:
        for opname, _ in OPS:
            for count in counts:
                for storage in STORAGES if count != MANY_BLOCKS else ("heap", "pageable"):
                    layout = F.LAYOUTS[i % 4]
                    inplace = i % 3 == 1
                    i += 1
                    if count == MANY_BLOCKS:
                        assert Wd.lib.b200mpi_set_param(b"own_block_bytes", 4096) == 0
                    done += loc_call(Wd, dn, opname, count, storage, layout, inplace, facade=i % 2 == 0)
                    if count == MANY_BLOCKS:
                        assert Wd.lib.b200mpi_set_param(b"own_block_bytes", 1 << 20) == 0
    for root in range(n):
        for k, dn in enumerate(DNS):
            for count in (1, 255, 4099):
                i += 1
                storage = STORAGES[i % 4]
                done += loc_call(Wd, dn, OPS[i % 2][0], count, storage, F.LAYOUTS[i % 4], inplace=(i % 5 == 0), root=root,
                                 facade=i % 3 == 0, null_recv=i % 2 == 0)
    mpi.Barrier()
    return {"checked": done}


def scenario_loc_capped(a):
    """Grids capped at 1 and 3 CTAs, so that every CTA makes several passes, aligned and at 8 mod 16."""
    Wd = World()
    done = 0
    for cap in (1, 3):
        assert Wd.lib.b200mpi_set_max_blocks(cap) == 0
        for j, dn in enumerate(DNS):
            for layout in ("aligned", "mixed"):
                done += loc_call(Wd, dn, OPS[j % 2][0], 20011, "heap", layout, inplace=j == 1)
            done += loc_call(Wd, dn, OPS[(j + 1) % 2][0], 9001, "heap", "split", root=Wd.n - 1, null_recv=True)
    assert Wd.lib.b200mpi_set_max_blocks(0) == 0
    mpi.Barrier()
    return {"checked": done}


def scenario_loc_mismatch(a):
    """Ranks that disagree end the call as B200MPI_ERR_PEER on every rank with send and recv untouched:
    AllreduceLoc against a two-shot Allreduce of the same bytes, AllreduceLoc against ReduceLoc, and a
    different op, dtype, count or root.  The next call works."""
    Wd = World()
    lib, rank, n = Wd.lib, Wd.rank, Wd.n
    odd = rank == 1
    count = 1000
    dt = R.LOC["f64"]
    xs = R.tie_heavy("f64", n, count, 55)
    done = 0
    for storage in ("heap", "pageable"):
        mk = L.DEVICE if storage == "heap" else L.HOST
        cases = (
            ("allreduce against allreduce_loc", lambda s, r: lib.b200mpi_allreduce(s, r, 2 * count, L.F64, L.MAX, mk) if odd
             else lib.b200mpi_allreduce_loc(s, r, count, L.F64, L.MAX, mk)),
            ("allreduce_loc against reduce_loc", lambda s, r: lib.b200mpi_reduce_loc(s, r, count, L.F64, L.MAX, 0, mk) if odd
             else lib.b200mpi_allreduce_loc(s, r, count, L.F64, L.MAX, mk)),
            ("different op", lambda s, r: lib.b200mpi_allreduce_loc(s, r, count, L.F64, L.MIN if odd else L.MAX, mk)),
            ("different dtype", lambda s, r: lib.b200mpi_allreduce_loc(s, r, count, L.I64 if odd else L.F64, L.MAX, mk)),
            ("different count", lambda s, r: lib.b200mpi_allreduce_loc(s, r, count - 1 if odd else count, L.F64, L.MAX, mk)),
            ("different root", lambda s, r: lib.b200mpi_reduce_loc(s, r, count, L.F64, L.MIN, 1 if odd else 0, mk)),
        )
        lib.b200mpi_set_algo(L.COLL_ALLREDUCE, L.ALGO_TWOSHOT)  # the plain Allreduce takes a barrier, not the LL path
        for name, call in cases:
            c = Wd.next_call()
            send = K.Buf(storage, dt, count, 0, rank, c, body=xs[rank])
            recv = K.Buf(storage, dt, count, 0, rank, c + 1)
            rc = call(send.ptr(), recv.ptr())
            assert rc == L.ERR_PEER, (name, storage, rc, L.last_error())
            F.check(send, "%s (%s): send untouched" % (name, storage))
            F.check(recv, "%s (%s): recv untouched" % (name, storage))
            send.free()
            recv.free()
            done += 1
        lib.b200mpi_set_algo(L.COLL_ALLREDUCE, 0)
        done += loc_call(Wd, "f64", "minloc", count, storage, "aligned")  # and the world still works
    mpi.Barrier()
    return {"checked": done}


def scenario_loc_wrap(a):
    """AllreduceLoc and ReduceLoc call after call across the scrub that ends on epoch 0 (the world
    starts a few launches below it).  Reports the epoch before and after."""
    Wd = World()
    first = L.get_param("epoch")
    done = 0
    for i in range(12):
        dn = DNS[i % 3]
        root = None if i % 2 == 0 else i % Wd.n
        done += loc_call(Wd, dn, OPS[i % 2][0], (257, 4099, 1)[i % 3], "heap" if i % 4 != 3 else "pinned", F.LAYOUTS[i % 4], root=root)
    mpi.Barrier()
    return {"checked": done, "epoch_first": first, "epoch_last": L.get_param("epoch")}


def scenario_loc_large(a):
    """64 MiB of pairs per rank: MINLOC of f64 and MAXLOC of f32 into every rank, then MAXLOC of i64 to
    the last rank, checked byte for byte against the oracle."""
    Wd = World()
    rank, n = Wd.rank, Wd.n
    count = (64 << 20) // 16
    done = 0
    for dn, opname, root in (("f64", "minloc", None), ("f32", "maxloc", None), ("i64", "maxloc", n - 1)):
        op = dict(OPS)[opname]
        ins = R.tie_heavy(dn, n, count, 9000 + len(dn) + op)
        send = mpi.Alloc(count, R.LOC[dn]).copy_from_host(ins[rank])
        recv = mpi.Alloc(count, R.LOC[dn])
        if root is None:
            mpi.AllreduceLoc(send, recv, op)
        else:
            mpi.ReduceLoc(send, recv, op, root)
        if root is None or rank == root:
            assert R.same(recv.to_host(), LO.allreduce_loc(ins, op)), "large %s %s" % (dn, opname)
        send.free()
        recv.free()
        done += 1
    mpi.Barrier()
    return {"checked": done}


def scenario_loc_best_point(a):
    """The use case: every rank holds a candidate point and its objective; MINLOC over (objective,
    loc = rank) names the rank with the best point (the lower rank on a tie), and a Bcast from it
    delivers that point to everyone.  Ranks 0 and n-1 share the worst value, the best one is held by
    two middle ranks (or rank 0 in a world of one)."""
    rank, n = mpi.Rank(), mpi.Size()
    objective = lambda r: 1.0 if r in (n // 2, n // 2 + 1) else 5.0 + (r % 3)  # noqa: E731
    point = lambda r: np.arange(6, dtype=np.float64) * (r + 1) - r  # noqa: E731
    mine = R.pairs(mpi.LOC_F64, [objective(rank)], [rank])
    best = np.zeros(1, mpi.LOC_F64)
    mpi.AllreduceLoc(mine, best, mpi.MIN)
    want_rank = min(range(n), key=lambda r: (objective(r), r))
    assert int(best["loc"][0]) == want_rank and float(best["val"][0]) == objective(want_rank), (best, want_rank)
    x = mpi.Alloc(6, np.float64).copy_from_host(point(rank))
    mpi.Bcast(x, int(best["loc"][0]))
    W.check_equal(x.to_host(), point(want_rank), "best point from rank %d" % want_rank)
    x.free()
    worst = np.zeros(1, mpi.LOC_F64)
    mpi.ReduceLoc(mine, worst if rank == 0 else None, mpi.MAX, 0)
    if rank == 0:
        want_worst = min(range(n), key=lambda r: (-objective(r), r))
        assert int(worst["loc"][0]) == want_worst, (worst, want_worst)
    mpi.Barrier()
    return {"checked": 2}


def scenario_loc_control_only(a):
    """Control plane only: both calls refuse with B200MPI_ERR_NO_DEVICE, through the C ABI and the facade."""
    lib = L.load()
    x, y = np.zeros(4, mpi.LOC_F64), np.zeros(4, mpi.LOC_F64)
    assert lib.b200mpi_allreduce_loc(x.ctypes.data, y.ctypes.data, 4, L.F64, L.MAX, L.HOST) == L.ERR_NO_DEVICE
    assert lib.b200mpi_reduce_loc(x.ctypes.data, y.ctypes.data, 4, L.F64, L.MIN, 0, L.HOST) == L.ERR_NO_DEVICE
    for call in (lambda: mpi.AllreduceLoc(x, y), lambda: mpi.ReduceLoc(x, y, mpi.MIN, 0)):
        try:
            call()
            raise AssertionError("data call succeeded without a device")
        except mpi.MpiError as e:
            if e.code != L.ERR_NO_DEVICE:
                raise
    return {"checked": 4}


W.SCENARIOS.update({k[len("scenario_"):]: v for k, v in list(globals().items()) if k.startswith("scenario_")})

if __name__ == "__main__":
    W.main()
