"""One rank of a test world for Alltoallv.  Usage as _worker.py: _alltoallv_worker.py <scenario>
--out FILE [scenario args] -mpi-* flags.  The scenarios drive the product through the public
mpi_b200 API / C ABI and check every result bit for bit against the numpy restatement
(_alltoallv_ref.py, test infrastructure only); the rest (argument parsing, Init, result file) is
_worker.py's."""
import ctypes
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _alltoallv_ref as A  # noqa: E402
import _worker as W  # noqa: E402
from _gather_worker import GDTYPES, gfill, sentinel  # noqa: E402
from _worker import L, O, SEED, check_equal, free_buffer, make_buffer, read_buffer, mpi  # noqa: E402


def sends_for(dt, m, salt):
    """Every rank's send buffer of the call described by m (each rank builds all of them to know
    what it must receive)."""
    return [gfill(dt, SEED + 31 * i + salt, sum(m[i])) for i in range(len(m))]


def check_call(kind, dt, m, what, salt=0):
    """One Alltoallv of the matrix m through the facade; recv against the restatement, send untouched.
    A uniform matrix also runs Alltoall, whose result must be the same bytes."""
    rank, n = mpi.Rank(), mpi.Size()
    sends = sends_for(dt, m, salt)
    scounts, rcounts = A.row(m, rank), A.col(m, rank)
    want = A.alltoallv(sends, m, rank)
    send = make_buffer(kind, sends[rank])
    recv = make_buffer(kind, sentinel(dt, sum(rcounts)))
    got, counts = mpi.Alltoallv(send, scounts, recv, rcounts)
    assert counts == rcounts, (counts, rcounts)
    check_equal(read_buffer(got), want, "alltoallv %s %s %s" % (what, kind, np.dtype(dt).name))
    check_equal(read_buffer(send), sends[rank], "alltoallv %s %s: send untouched" % (what, kind))
    done = 1
    if len({c for r in m for c in r}) == 1 and n > 0:
        fixed = make_buffer(kind, sentinel(dt, sum(rcounts)))
        mpi.Alltoall(send, fixed)
        check_equal(read_buffer(fixed), read_buffer(got), "alltoall == alltoallv %s %s" % (kind, np.dtype(dt).name))
        check_equal(read_buffer(fixed), O.alltoall([s.reshape(-1) for s in sends], rank), "alltoall oracle %s" % kind)
        free_buffer(fixed)
        done += 1
    free_buffer(send)
    free_buffer(recv)
    return done


def scenario_alltoallv(a):
    """Every table of _alltoallv_ref.tables over the dtypes and memory kinds."""
    n = mpi.Size()
    done = 0
    for kind in a.kinds.split(","):
        for dn in a.dtypes.split(","):
            for name, m in A.tables(n, SEED + n):
                done += check_call(kind, GDTYPES[dn], m, name)
    if n == 1:  # a world of one still checks its table: send_counts[0] must equal recv_counts[0]
        lib = L.load()
        x, y = np.arange(4, dtype=np.float32), np.full(8, -7, dtype=np.float32)
        rc = lib.b200mpi_alltoallv(x.ctypes.data, (ctypes.c_size_t * 1)(4), y.ctypes.data, (ctypes.c_size_t * 1)(5), L.F32, L.HOST)
        assert rc == L.ERR_PEER, (rc, L.last_error())
        check_equal(y, np.full(8, -7, dtype=np.float32), "world of one mismatch: recv untouched")
        done += 1
    mpi.Barrier()
    return {"checked": done}


def scenario_alltoallv_unaligned(a):
    """Heap offsets that are not 16-byte aligned and differ between ranks (odd element offsets for
    bytes, 4/8-byte offsets for the wider types), with uniform 16-byte-multiple blocks (ranks then
    pick different access widths for the same call) and odd random blocks."""
    rank, n = mpi.Rank(), mpi.Size()
    rng = np.random.default_rng(SEED + 7 * n)
    done = 0
    for dn, dt in GDTYPES.items():
        for name, m in (("uniform 4096", [[4096] * n for _ in range(n)]),
                        ("odd", [[2 * int(rng.integers(0, 600)) + 1 for _ in range(n)] for _ in range(n)])):
            sends = sends_for(dt, m, 3)
            scounts, rcounts = A.row(m, rank), A.col(m, rank)
            so, ro = 1 + rank % 3, 1 + (rank + 1) % 2
            sbig, rbig = mpi.Alloc(sum(scounts) + 8, dt), mpi.Alloc(sum(rcounts) + 8, dt)
            send = sbig[so:so + sum(scounts)].copy_from_host(sends[rank])
            recv = rbig[ro:ro + sum(rcounts)].copy_from_host(sentinel(dt, sum(rcounts)))
            mpi.Alltoallv(send, scounts, recv, rcounts)
            check_equal(recv.to_host(), A.alltoallv(sends, m, rank), "unaligned alltoallv %s %s" % (dn, name))
            check_equal(send.to_host(), sends[rank], "unaligned alltoallv %s %s: send untouched" % (dn, name))
            sbig.free()
            rbig.free()
            done += 1
    mpi.Barrier()
    return {"checked": done}


def scenario_alltoallv_mismatch(a):
    """Tables that disagree (one recv count off by one, two entries of a row swapped), a dtype
    disagreement, and a rank that calls Alltoall while the others call Alltoallv: B200MPI_ERR_PEER
    on every rank, buffers untouched (heap and host), and the next Alltoallv works."""
    rank, n = mpi.Rank(), mpi.Size()
    lib = L.load()
    m = [[3 + 5 * i + 2 * j for j in range(n)] for i in range(n)]  # entries of a row all differ
    cap = 2 * max(sum(r) for r in m) + 64  # room for the i64 view of the dtype disagreement
    done = 0
    for kind in ("heap", "host"):
        mk = L.DEVICE if kind == "heap" else L.HOST
        x = make_buffer(kind, gfill(np.float32, SEED + rank, cap))
        y = make_buffer(kind, sentinel(np.float32, cap))
        xp = x.ptr if kind == "heap" else x.ctypes.data
        yp = y.ptr if kind == "heap" else y.ctypes.data
        srow, rcol = A.row(m, rank), A.col(m, rank)
        off_by_one, swapped = list(rcol), list(srow)
        off_by_one[0] += 1
        swapped[0], swapped[1] = swapped[1], swapped[0]
        st = lambda t: (ctypes.c_size_t * n)(*t)  # noqa: E731
        cases = (
            ("recv count off by one", lambda: lib.b200mpi_alltoallv(xp, st(srow), yp, st(off_by_one if rank == 1 else rcol), L.F32, mk)),
            ("row entries swapped", lambda: lib.b200mpi_alltoallv(xp, st(swapped if rank == 1 else srow), yp, st(rcol), L.F32, mk)),
            ("dtype disagreement", lambda: lib.b200mpi_alltoallv(xp, st(srow), yp, st(rcol), L.I64 if rank == 1 else L.F32, mk)),
            ("alltoall against alltoallv", lambda: (lib.b200mpi_alltoall(xp, yp, 3, L.F32, mk) if rank == 1 else
                                                    lib.b200mpi_alltoallv(xp, st(srow), yp, st(rcol), L.F32, mk))),
        )
        for name, call in cases:
            rc = call()
            assert rc == L.ERR_PEER, (name, kind, rc, L.last_error())
            # The fixed-count Alltoall copies a staged host result back whether or not the call
            # succeeded, so only that rank's host recv is exempt from the check.
            if not (name.startswith("alltoall against") and rank == 1 and kind == "host"):
                check_equal(read_buffer(y), sentinel(np.float32, cap), "%s %s: recv untouched" % (name, kind))
            check_equal(read_buffer(x), gfill(np.float32, SEED + rank, cap), "%s %s: send untouched" % (name, kind))
            done += 1
            # and the world still works
            sends = sends_for(np.float32, m, 11)
            if kind == "host":
                y[:] = sentinel(np.float32, cap)
            send = make_buffer(kind, sends[rank])
            got, _ = mpi.Alltoallv(send, srow, y[:sum(rcol)], rcol)
            check_equal(read_buffer(got), A.alltoallv(sends, m, rank), "alltoallv after %s (%s)" % (name, kind))
            free_buffer(send)
            if kind == "heap":
                y.copy_from_host(sentinel(np.float32, cap))
            else:
                y[:] = sentinel(np.float32, cap)
            done += 1
        free_buffer(x)
        free_buffer(y)
    mpi.Barrier()
    return {"checked": done}


def scenario_alltoallv_strings(a):
    """u8 strings of a different length for every (source, destination) pair, with the recv counts
    learnt by the facade; the receiver splits the packed bytes with the returned counts."""
    rank, n = mpi.Rank(), mpi.Size()
    words = [['"%d to %d%s"' % (i, j, "!" * (3 * i + j)) for j in range(n)] for i in range(n)]
    send = "".join(words[rank]).encode()
    counts = [len(w.encode()) for w in words[rank]]
    got, learnt = mpi.Alltoallv(send, counts)
    assert learnt == [len(words[k][rank].encode()) for k in range(n)], learnt
    parts, lo = [], 0
    for c in learnt:
        parts.append(got[lo:lo + c].tobytes().decode())
        lo += c
    assert parts == [words[k][rank] for k in range(n)], parts
    # a recv that is too small is replaced, one that is larger is used through a view
    got, _ = mpi.Alltoallv(send, counts, np.zeros(2, dtype=np.uint8))
    assert got.tobytes().decode() == "".join(words[k][rank] for k in range(n))
    big = np.full(4096, 7, dtype=np.uint8)
    got, _ = mpi.Alltoallv(send, counts, big, learnt)
    assert got.size == sum(learnt) and got.tobytes().decode() == "".join(words[k][rank] for k in range(n)) and big[sum(learnt)] == 7
    mpi.Barrier()
    return {"checked": 3}


def scenario_alltoallv_large(a):
    """About 64 MiB of f32 per rank on a skewed table: three quarters of every rank's send goes to
    its right neighbour, the rest in odd-sized blocks to the others.  Bit-exact."""
    rank, n = mpi.Rank(), mpi.Size()
    big, rest = 12 << 20, (4 << 20) // max(n - 1, 1)
    m = [[big if j == (i + 1) % n else rest + 2 * j + 1 for j in range(n)] for i in range(n)]
    sends = [O.fill(np.float32, SEED + i, sum(m[i])) for i in range(n)]
    scounts, rcounts = A.row(m, rank), A.col(m, rank)
    send = mpi.Alloc(sum(scounts), np.float32).copy_from_host(sends[rank])
    recv = mpi.Alloc(sum(rcounts), np.float32)
    mpi.Alltoallv(send, scounts, recv, rcounts)
    check_equal(recv.to_host(), A.alltoallv(sends, m, rank), "alltoallv 64 MiB skewed")
    send.free()
    recv.free()
    mpi.Barrier()
    return {"checked": 1}


def scenario_alltoallv_control_only(a):
    """Control plane only: Alltoallv refuses with B200MPI_ERR_NO_DEVICE, through the C ABI and the facade."""
    n = mpi.Size()
    lib = L.load()
    x = np.zeros(4 * n, dtype=np.float32)
    y = np.zeros(4 * n, dtype=np.float32)
    tab = (ctypes.c_size_t * n)(*([4] * n))
    rc = lib.b200mpi_alltoallv(x.ctypes.data, tab, y.ctypes.data, tab, L.F32, L.HOST)
    assert rc == L.ERR_NO_DEVICE, rc
    for call in (lambda: mpi.Alltoallv(x, [4] * n, y, [4] * n), lambda: mpi.Alltoallv(x, [4] * n)):
        try:
            call()
            raise AssertionError("data call succeeded without a device")
        except mpi.MpiError as e:
            if e.code != L.ERR_NO_DEVICE:
                raise
    return {"checked": 3}


W.SCENARIOS.update({k[len("scenario_"):]: v for k, v in list(globals().items()) if k.startswith("scenario_")})

if __name__ == "__main__":
    W.main()
